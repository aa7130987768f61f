"""MuZeroModelMLP's tensor-core layers (model kind 4) against float64, each on its own inputs (the kernel's output of the layer
before, lz_model_debug_net_stage), with the bounds of test_gpu_mlp_ez_layers.py: |y - y64| <= 2^-17 M + 2^-23 (M the
magnitude sum of the layer) in tc3, and beyond it in tc1 -- a dropped hi / lo pass would fail.  The three heads (hidden
layer + FC2 pieces) are bounded through the magnitude of both Linears; the reward head reads fc_dynamics_2's output (or
fc_dynamics' without res_connection_in_dynamics)."""
import pytest
import torch

import mlp_mz_model_ref as MR
from test_gpu_mlp_ez_layers import layer_refs, linear
from test_gpu_mlp_mz import inputs, make
from test_gpu_net_layers import worst

pytestmark = pytest.mark.gpu

TAU, ALPHA = 2.0 ** -17, 2.0 ** -23
B = 129


def stage(cu, which, x, action, s):
    from lightzero_b200 import cabi
    L, K, A = cu.latent_state_dim, cu.value_support_size, cu.action_space_size
    n = x.shape[0]
    out = torch.zeros(n * (2 * K + A + 2 + 2 * L), device="cuda")
    info = (cabi.ctypes.c_int32 * 8)()
    cabi.check(cu._lib.lz_model_debug_net_stage(cu._h, which, n, x.contiguous().data_ptr(), action.data_ptr(), s, out.data_ptr(),
                                                out.numel() * 4, info, cabi.stream_ptr()), "lz_model_debug_net_stage")
    torch.cuda.synchronize()
    D = info[7]
    if s < D:
        return out[:n * L].view(n, L).double().cpu(), list(info)
    v = out.cpu().double()[2 * n * L:]
    o = dict(value=v[:n * K].view(n, K), policy=v[n * K:n * (K + A)].view(n, A))
    if not which:
        o["reward"] = v[n * (K + A + 1):n * (2 * K + A + 1)].view(n, K)
    return o, list(info)


def head(mlp, x):
    """float64 MLP_V2 head (Linear + BN + ReLU, Linear) on x and the magnitude bound of both Linears"""
    hdn, M1 = linear(mlp[0], mlp[1], x, act="relu")
    y, M = linear(mlp[3], None, hdn)
    return y, M + mlp[3].weight.double().abs().matmul(M1.T).T


def ratios(name, ref, cu, which):
    """{layer: worst |err| / bound} of one program, and the launch info of the whole program (R, CTAs, last, layers, passes,
    shared memory, ring stages, dense layers)"""
    A, res = MR.CONFIGS[name][1], MR.CONFIGS[name][3]
    obs, action = inputs(name, B, 77)
    action = action.to(torch.int32).cuda()
    x0 = obs.double() if which else cu.initial_inference(obs.cuda()).latent_state.double().cpu()
    onehot = torch.nn.functional.one_hot(action.long().cpu(), A).double()
    layers = layer_refs(ref, which)
    D = len(layers)
    prev, z, dumps, r = x0, x0, [], {}
    for s, (lin, bn, act, oh, resid, ln) in enumerate(layers):
        got, info = stage(cu, which, x0.float().cuda(), action, s)
        assert info[7] == D
        if res and not which and s == 4:
            prev = dumps[1]             # the prediction network reads next = fc_dynamics_1 + latent, not fc_dynamics_2's output
        y, M = linear(lin, bn, prev, onehot if oh else None, act)
        if resid:
            y, M = y + z, M + z.abs()
        if ln is not None:      # first order: the error of v passes through rstd * |w|; mean / variance shifts add its row mean
            mean, var = y.mean(1, keepdim=True), y.var(1, unbiased=False, keepdim=True)
            rstd = 1.0 / torch.sqrt(var + 1e-5)
            M = rstd * ln.weight.double().abs() * (M + M.mean(1, keepdim=True))
            y = (y - mean) * rstd * ln.weight.double() + ln.bias.double()
        r[f"L{s}"] = worst(got - y, TAU * M + ALPHA)
        prev = got
        dumps.append(got)
    whole, info = stage(cu, which, x0.float().cuda(), action, D)
    P = ref.prediction_network
    heads = [("value", P.fc_value_head, prev), ("policy", P.fc_policy_head, prev)]
    if not which:
        heads.append(("reward", ref.dynamics_network.fc_reward_head, dumps[3] if res else dumps[1]))
    for key, mlp, x in heads:
        y, M = head(mlp, x)
        r[key] = worst(whole[key] - y, TAU * M + ALPHA)
    return r, info


@pytest.mark.parametrize("name", list(MR.CONFIGS))
@pytest.mark.parametrize("which", [1, 0], ids=["initial", "recurrent"])
def test_layers_match_float64_and_tc1_fails(name, which):
    ref, cu = make(name, 21)
    r3, info = ratios(name, ref, cu, which)
    print(f"\n[mlp-mz-layers] {name} NC={cu.latent_state_dim // 32} which={which} layers={info[3]} tc3 "
          + " ".join(f"{k}={v:.3g}" for k, v in r3.items()))
    assert all(v <= 1.0 for v in r3.values()), r3
    assert which or "reward" in r3
    if name == "l32_a608" and not which:
        assert info[3] == 66            # the longest program the kernel takes (kMezMaxLayers)
    cu.set_math("tc1")                  # a math mode: the tensor-core kernel, not the fp32 one
    r1, _ = ratios(name, ref, cu, which)
    print(f"[mlp-mz-layers] {name} which={which} tc1 " + " ".join(f"{k}={v:.3g}" for k, v in r1.items()))
    assert all(v > 1.0 for v in r1.values()), r1
