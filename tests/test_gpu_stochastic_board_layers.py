"""The board Stochastic MuZero network (StochasticMuZeroModel, downsample=False) on k_board_tc, layer by layer against float64
(lz_model_debug_net_stage): `init` (which 1: representation + prediction), `rec` (which 0: dynamics over [afterstate | chance
plane] + prediction) and `after` (which 2: afterstate dynamics over [latent | action plane] + afterstate prediction, policy
chance_space_size wide).

Each 3x3 layer's float64 reference runs on the operands the kernel consumed, with the bound of test_gpu_board_layers.py:
|y_cuda - y_f64| <= TAU * M + ALPHA * S, TAU = 2^-17; 3xFP16 must stay under a quarter of it and a single fp16 pass (tc1) must
exceed it by >= 8x on every 3x3 layer.  The dynamics convs' encoding plane enters the reference as the float32 value
option / n the reference computes.  Each head is compared on the unsplit hook output under its first-order bound
(C + hc * P + hid + 8) * 2^-24."""
import copy

import pytest
import torch

import stoch_board_model_ref as SB
from test_gpu_net_layers import ALPHA, TAU, check_scalars, head_reference, layer_reference, split_full, split_hi_lo, worst

pytestmark = pytest.mark.gpu

NAMES = list(SB.CONFIGS)
U32 = 2.0 ** -24
B = 37


def make(name, math):
    import lightzero_b200 as lzb
    ref = SB.build(name, NAMES.index(name))
    cu = lzb.StochasticMuZeroModel(**SB.model_kwargs(name)).load_state_dict(ref.state_dict())
    cu.set_math(math)
    return copy.deepcopy(ref).double().cuda().eval(), cu


def stage(cu, which, x, option, s, nl):
    """(f32 output, h_info) of program `which` cut after layer `s` (s == nl: the whole program)"""
    import numpy as np
    from lightzero_b200 import cabi
    n, K = x.shape[0], cu.value_support_size
    P = cu.chance_space_size if which == 2 else cu.action_space_size
    C, H, W = cu.latent_shape
    size = n * C * H * W if s < nl else n * (2 * K + 2 * P + 4)
    buf = torch.full((size,), float("nan"), dtype=torch.float32, device="cuda")
    info = np.zeros(8, np.int32)
    opt = option.to(torch.int32).contiguous() if option is not None else None
    cabi.check(cu._lib.lz_model_debug_net_stage(cu._h, which, n, x.contiguous().data_ptr(), cabi.ptr(opt), s, buf.data_ptr(),
                                                buf.numel() * 4, info.ctypes.data, cabi.stream_ptr()), "lz_model_debug_net_stage")
    torch.cuda.synchronize()
    return buf, [int(v) for v in info]


def program(ref64, which):
    """[(conv, bn, kind)] of a program, its reward head's hook layer, and its (reward, value, policy) head modules"""
    rep = ref64.representation_network
    dyn, pred = ((ref64.afterstate_dynamics_network, ref64.afterstate_prediction_network) if which == 2 else
                 (ref64.dynamics_network, ref64.prediction_network))
    if which == 1:
        layers, blocks = [(rep.conv, rep.norm, "rep")], list(rep.resblocks) + list(pred.resblocks)
    else:
        layers, blocks = [(dyn.conv, dyn.bn, "dyn")], list(dyn.resblocks) + list(pred.resblocks)
    for b in blocks:
        layers += [(b.conv1[0], b.conv1[1], "conv1"), (b.conv2[0], b.conv2[1], "conv2")]
    vbn, pbn = (pred.bn_value, pred.bn_policy) if which == 2 else (pred.norm_value, pred.norm_policy)
    heads = dict(value=(pred.conv1x1_value, vbn, pred.fc_value), policy=(pred.conv1x1_policy, pbn, pred.fc_policy))
    if which != 1:
        heads["reward"] = (dyn.conv1x1_reward, dyn.bn_reward, dyn.fc_reward_head)
    return layers, 2 * len(dyn.resblocks), heads


def run_program(cu, ref64, which, x0, option):
    layers, rew_hook, heads = program(ref64, which)
    nl, n = len(layers), x0.shape[0]
    C, H, W = cu.latent_shape
    P = cu.chance_space_size if which == 2 else cu.action_space_size
    dumps, infos = [], []
    for L in range(nl):
        buf, info = stage(cu, which, x0, option, L, nl)
        dumps.append(buf.view(n, C, H, W).double())
        infos.append(info)
    buf, info = stage(cu, which, x0, option, nl, nl)
    infos.append(info)
    out = split_full(buf, n, cu.value_support_size, P, 0)
    x64 = x0.double()
    plane = None
    if which != 1:
        N = cu.action_space_size if which == 2 else cu.chance_space_size
        plane = (option.float().view(n, 1, 1, 1) * torch.ones(n, 1, H, W, device="cuda") / N).double()
    ratios = {}
    with torch.no_grad():
        for L, (conv, bn, kind) in enumerate(layers):
            res = x64 if kind == "dyn" else (dumps[L - 2] if kind == "conv2" else None)
            y, M, S = layer_reference(conv, bn, kind, split_hi_lo(dumps[L - 1] if L else x64), res, plane)
            ratios[f"L{L}:{kind}"] = worst(dumps[L] - y, TAU["conv1"] * M + ALPHA * S)
        for name, (conv, bn, mlp) in heads.items():
            x = dumps[rew_hook] if name == "reward" else dumps[nl - 1]
            y, M, S = head_reference(conv, bn, mlp, x)
            tau = (C + conv.out_channels * H * W + mlp[0].out_features + 8) * U32
            ratios[f"{name} head"] = worst(out[f"{name}_logits"].double() - y, tau * M + ALPHA * S)
    return ratios, out, infos


def inputs(cu, name):
    obs_shape, A, NC = SB.CONFIGS[name][:3]
    g = torch.Generator().manual_seed(100 + NAMES.index(name))
    obs = torch.rand((B,) + tuple(obs_shape), generator=g).cuda()
    action, chance = torch.randint(0, A, (B,), generator=g).cuda(), torch.randint(0, NC, (B,), generator=g).cuda()
    latent = cu.initial_inference(obs).latent_state
    after = cu.recurrent_inference(latent, action, False).latent_state
    return {1: (obs, None), 2: (latent, action), 0: (after, chance)}


@pytest.mark.parametrize("name", NAMES)
def test_layers_match_float64_and_tc1_fails(name):
    ref64, cu = make(name, "tc3")
    progs = inputs(cu, name)
    for math in ("tc3", "tc1"):
        cu.set_math(math)
        for which, (x0, option) in progs.items():
            ratios, out, infos = run_program(cu, ref64, which, x0, option)
            print(f"\n[stoch-board-layers] {name} {math} program {which}: " + " ".join(f"{k}={v:.3g}" for k, v in ratios.items()))
            assert all(info[5] == (3 if math == "tc3" else 1) for info in infos), infos
            if math == "tc1":
                weak = {k: r for k, r in ratios.items() if k.startswith("L") and not r >= 8.0}
                assert not weak, f"{name} program {which}: tc1 within 8x of the bound on {weak}"
                continue
            bad = {k: r for k, r in ratios.items() if not r <= (0.25 if k.startswith("L") else 1.0)}
            assert not bad, f"{name} program {which}: over the bound {bad}"
            assert all(r > 0 for k, r in ratios.items() if k.endswith("head")), ratios   # an exact head is a dead one
            check_scalars(out, 0 if which != 1 else 1, False, SB.CONFIGS[name][7])


def test_after_stage_refused_by_muzero_board_model():
    """which 2 is the Stochastic MuZero models' afterstate program: a MuZero board model refuses it"""
    import board_model_ref as BR
    import lightzero_b200 as lzb
    from lightzero_b200 import cabi
    cu = lzb.MuZeroModel(**BR.model_kwargs("tictactoe")).load_state_dict(BR.build("tictactoe", 0).state_dict())
    x, a = torch.zeros(2, 16, 3, 3, device="cuda"), torch.zeros(2, dtype=torch.int32, device="cuda")
    buf, info = torch.zeros(4096, device="cuda"), (cabi.ctypes.c_int32 * 8)()
    with pytest.raises(cabi.LzError, match="which 2"):
        cabi.check(cu._lib.lz_model_debug_net_stage(cu._h, 2, 2, x.data_ptr(), a.data_ptr(), 0, buf.data_ptr(), buf.numel() * 4,
                                                    info, cabi.stream_ptr()), "lz_model_debug_net_stage")
