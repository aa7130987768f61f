"""EfficientZeroModelMLP's tensor-core layers against float64, each on its own inputs (the kernel's output of the layer before,
lz_model_debug_net_stage): |y - y64| <= 2^-17 M + 2^-23 (test_gpu_net_layers.py's bound, M the magnitude sum of the layer) in
tc3, and beyond it in tc1 -- a dropped hi / lo pass would fail.  The LayerNorm layer is bounded to first order through its
rstd, the heads (hidden layer + FC2 pieces) through the magnitude of both Linears, and the LSTM on this model's own features
by test_gpu_ez_oracle.py's lstm_bound."""
import pytest
import torch

import mlp_ez_model_ref as MR
from test_gpu_ez_oracle import TAU_LSTM
from test_gpu_mlp_ez import inputs, make
from test_gpu_net_layers import lstm_bound, worst

pytestmark = pytest.mark.gpu

TAU, ALPHA = 2.0 ** -17, 2.0 ** -23
B = 129


def stage(cu, which, x, action, s):
    from lightzero_b200 import cabi
    L, K, A = cu.latent_state_dim, cu.value_support_size, cu.action_space_size
    n = x.shape[0]
    out = torch.zeros(n * (K + A + 1 + 2 * L), device="cuda")
    info = (cabi.ctypes.c_int32 * 8)()
    cabi.check(cu._lib.lz_model_debug_net_stage(cu._h, which, n, x.contiguous().data_ptr(), action.data_ptr(), s, out.data_ptr(),
                                                out.numel() * 4, info, cabi.stream_ptr()), "lz_model_debug_net_stage")
    torch.cuda.synchronize()
    D = info[7]
    if s < D:
        return out[:n * L].view(n, L).double().cpu(), D
    o = out.cpu().double()
    v = o[2 * n * L:]
    return dict(feat=o[n * L:2 * n * L].view(n, L), value=v[:n * K].view(n, K), policy=v[n * K:n * (K + A)].view(n, A)), D


def linear(lin, bn, x, xa=None, act=None):
    """float64 Linear (+ BN) on x and its magnitude sum M; xa: one-hot columns appended to x"""
    W, b = lin.weight.double(), lin.bias.double()
    xin = x if xa is None else torch.cat([x, xa], 1)
    y, M = xin @ W.T + b, xin.abs() @ W.abs().T + b.abs()
    if bn is not None:
        s = bn.weight.double() / torch.sqrt(bn.running_var.double() + 1e-5)
        mu, beta = bn.running_mean.double(), bn.bias.double()
        y, M = s * (y - mu) + beta, s.abs() * (M + mu.abs()) + beta.abs()
    if act == "relu":
        y = torch.relu(y)
    elif act == "gelu":
        y, M = torch.nn.functional.gelu(y, approximate="tanh"), 1.13 * M
    return y, M


def layer_refs(ref, which):
    """(Linear, BN, activation, one-hot?, residual?, LayerNorm?) of the dense layers of a program, in program order"""
    R, D, P = ref.representation_network, ref.dynamics_network, ref.prediction_network
    pred = [(P.fc_prediction_common[0], P.fc_prediction_common[1], "relu", False, False, None),
            (P.fc_prediction_common[3], P.fc_prediction_common[4], "relu", False, False, None)]
    if which:
        return [(R.fc_representation[0], R.fc_representation[1], "gelu", False, False, None),
                (R.fc_representation[3], None, None, False, False, R.norm)] + pred
    if D.res_connection_in_dynamics:
        f1, f2 = D.fc_dynamics_1, D.fc_dynamics_2
        return [(f1[0], f1[1], "relu", True, False, None), (f1[3], f1[4], "relu", False, True, None),
                (f2[0], f2[1], "relu", False, False, None), (f2[3], f2[4], "relu", False, False, None)] + pred
    f = D.fc_dynamics
    return [(f[0], f[1], "relu", True, False, None), (f[3], f[4], "relu", False, False, None)] + pred


def ratios(ref, cu, which):
    obs_dim, A, L, H, res = MR.CONFIGS[NAME]
    obs, action, h0, c0 = inputs(NAME, B, 77)
    action = action.to(torch.int32).cuda()
    x0 = obs.double() if which else cu.initial_inference(obs.cuda()).latent_state.double().cpu()
    onehot = torch.nn.functional.one_hot(action.long().cpu(), A).double()
    prev, r = x0, {}
    layers = layer_refs(ref, which)
    D = len(layers)
    z, dumps = x0, []
    for s, (lin, bn, act, oh, resid, ln) in enumerate(layers):
        got, D2 = stage(cu, which, x0.float().cuda(), action, s)
        assert D2 == D
        if res and not which and s == 4:
            prev = dumps[1]             # the prediction network reads next = fc_dynamics_1 + latent, not the LSTM input
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
    whole, _ = stage(cu, which, x0.float().cuda(), action, D)
    P = ref.prediction_network
    for name, mlp in (("value", P.fc_value_head), ("policy", P.fc_policy_head)):
        hdn, M1 = linear(mlp[0], mlp[1], prev, act="relu")
        y, M = linear(mlp[3], None, hdn)
        M = M + mlp[3].weight.double().abs().matmul(M1.T).T
        r[name] = worst(whole[name] - y, TAU * M + ALPHA)
    if not which:
        feat = whole["feat"].cuda()
        dyn = ref.dynamics_network
        lstm = torch.nn.LSTM(L, H).double().cuda()
        lstm.load_state_dict(dyn.lstm.state_dict())
        h1, c1, eh, ec = lstm_bound(lstm, feat, h0[0].double().cuda(), c0[0].double().cuda(), tau=TAU_LSTM)
        lat = x0.float().cuda()
        o = cu.recurrent_inference(lat, (h0.cuda(), c0.cuda()), action)
        r["h"] = worst(o.reward_hidden_state[0][0].double() - h1, eh)
        r["c"] = worst(o.reward_hidden_state[1][0].double() - c1, ec)
    return r


NAME = None


@pytest.mark.parametrize("name", ["cartpole", "lunarlander", "minigrid", "l96_h48", "l32_o1", "l64_o4096", "l192"])
@pytest.mark.parametrize("which", [1, 0], ids=["initial", "recurrent"])
def test_layers_match_float64_and_tc1_fails(name, which):
    global NAME
    NAME = name
    ref, cu = make(name, 21)
    r3 = ratios(ref, cu, which)
    print(f"\n[mlp-ez-layers] {name} NC={cu.latent_state_dim // 32} which={which} tc3 " + " ".join(f"{k}={v:.3g}" for k, v in r3.items()))
    assert all(v <= 1.0 for v in r3.values()), r3
    cu.set_math("tc1")
    r1 = ratios(ref, cu, which)
    print(f"[mlp-ez-layers] {name} which={which} tc1 " + " ".join(f"{k}={v:.3g}" for k, v in r1.items()))
    wg = [k for k in r1 if k.startswith("L") or k in ("value", "policy")]
    assert all(r1[k] > 1.0 for k in wg), {k: r1[k] for k in wg}
