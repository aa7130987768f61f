"""The board-game network (k_board_tc, downsample=False) layer by layer against float64 (lz_model_debug_net_stage).

As in test_gpu_net_layers.py, the hook runs a copy of the recurrent program (dynamics conv, dynamics ResBlocks, prediction
ResBlocks, heads) or of the initial_inference program (representation conv on the observation planes, representation
ResBlocks, prediction ResBlocks, value / policy heads) cut off after one layer and returns that layer's fp32 output.  Each
layer's float64 reference runs on exactly the operands the kernel consumed: the previous dump (or the observation planes)
split into fp16 hi / lo as the MMA input, the unsplit fp32 dump as the ResBlock residual (the kernel keeps skips as fp32 rows),
and the layer is compared element by element with

    |y_cuda - y_f64| <= TAU * M + ALPHA * S

(M: the layer in float64 on absolute values, S: operands whose fp16 lo part can be subnormal; test_gpu_net_layers.layer_reference).
The 3x3 layers use that file's TAU of 2^-17 with its margins: 3xFP16 stays under a quarter of the bound (at most 0.12 measured
on an H100), a single fp16 pass (tc1) exceeds it by >= 8x on every 3x3 layer (at least 12x measured): a dropped hi/lo pass is
seen.

The heads run in fp32 FMA on the CUDA cores from the fp32 latent rows, so each head is compared on the unsplit hook output
with the first-order rounding bound of its chain of dot products: TAU_head = (C + hc * P + hid + 8) * 2^-24.  The scalars are
h^-1 of the softmax expectation of the kernel's own logits, bit-identical whether the raw logits are requested or not.
"""
import copy

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import board_model_ref as BR
from test_gpu_net_layers import ALPHA, TAU, check_scalars, head_reference, layer_reference, split_full, split_hi_lo, worst

pytestmark = pytest.mark.gpu

NAMES = list(BR.BOARD_CONFIGS)
U32 = 2.0 ** -24


def make(name, math, seed=21):
    import lightzero_b200 as lzb
    ref = BR.build(name, seed)
    cu = lzb.MuZeroModel(**BR.model_kwargs(name)).load_state_dict(ref.state_dict())
    cu.set_math(math)
    return copy.deepcopy(ref).double().cuda().eval(), cu


def board_stage(cu, which, x, action, stage, nl):
    """(f32 output, h_info) of the board program cut after layer `stage` (stage == nl: the whole program)"""
    from lightzero_b200 import cabi
    B, K, A = x.shape[0], cu.value_support_size, cu.action_space_size
    C, H, W = cu.latent_shape
    n = B * C * H * W if stage < nl else B * (2 * K + 2 * A + 4)
    buf = torch.full((n,), float("nan"), dtype=torch.float32, device="cuda")
    info = np.zeros(8, np.int32)
    act = action.to(torch.int32).contiguous() if action is not None else None
    cabi.check(cu._lib.lz_model_debug_net_stage(cu._h, which, B, x.contiguous().data_ptr(), cabi.ptr(act), stage, buf.data_ptr(),
                                                buf.numel() * 4, info.ctypes.data, cabi.stream_ptr()), "lz_model_debug_net_stage")
    torch.cuda.synchronize()
    return buf, [int(v) for v in info]


def program(ref64, which):
    """[(conv, bn, kind)] of the recurrent (0) or initial (1) board program, and the layer the reward head hooks"""
    dyn, pred, rep = ref64.dynamics_network, ref64.prediction_network, ref64.representation_network
    if which == 0:
        layers, blocks = [(dyn.conv, dyn.norm_common, "dyn")], list(dyn.resblocks) + list(pred.resblocks)
    else:
        layers, blocks = [(rep.conv, rep.norm, "rep")], list(rep.resblocks) + list(pred.resblocks)
    for b in blocks:
        layers += [(b.conv1[0], b.conv1[1], "conv1"), (b.conv2[0], b.conv2[1], "conv2")]
    return layers, (2 * len(dyn.resblocks) if which == 0 else None)


def run_program(cu, ref64, which, x0, action):
    """every layer and head of one program against float64: ({stage: worst |err| / bound}, full outputs, h_infos)"""
    layers, rew_hook = program(ref64, which)
    nl, B, A = len(layers), x0.shape[0], cu.action_space_size
    C, H, W = cu.latent_shape
    dumps, infos = [], []
    for L in range(nl):
        buf, info = board_stage(cu, which, x0, action, L, nl)
        dumps.append(buf.view(B, C, H, W).double())
        infos.append(info)
    buf, info = board_stage(cu, which, x0, action, nl, nl)
    infos.append(info)
    out = split_full(buf, B, cu.value_support_size, A, 0)
    x64 = x0.double()
    onehot = F.one_hot(action.long(), A).double().view(B, A, 1, 1).expand(B, A, H, W) if which == 0 else None
    ratios = {}
    with torch.no_grad():
        for L, (conv, bn, kind) in enumerate(layers):
            res = x64 if kind == "dyn" else (dumps[L - 2] if kind == "conv2" else None)
            y, M, S = layer_reference(conv, bn, kind, split_hi_lo(dumps[L - 1] if L else x64), res, onehot)
            ratios[f"L{L}:{kind}"] = worst(dumps[L] - y, TAU["conv1"] * M + ALPHA * S)
        pred, dyn = ref64.prediction_network, ref64.dynamics_network
        heads = [("value", pred.conv1x1_value, pred.norm_value, pred.fc_value, dumps[nl - 1], out["value_logits"]),
                 ("policy", pred.conv1x1_policy, pred.norm_policy, pred.fc_policy, dumps[nl - 1], out["policy_logits"])]
        if which == 0:
            heads.append(("reward", dyn.conv1x1_reward, dyn.norm_reward, dyn.fc_reward_head, dumps[rew_hook], out["reward_logits"]))
        for name, conv, bn, mlp, x, got in heads:
            y, M, S = head_reference(conv, bn, mlp, x)
            tau = (C + conv.out_channels * H * W + mlp[0].out_features + 8) * U32
            ratios[f"{name} head"] = worst(got.double() - y, tau * M + ALPHA * S)
    return ratios, out, infos


def inputs(cu, name, B, seed):
    """(observations, latents from the model's own initial_inference, actions)"""
    obs_shape, A = BR.config(name)[0], BR.config(name)[1]
    g = torch.Generator().manual_seed(seed)
    obs = torch.rand((B,) + tuple(obs_shape), generator=g).cuda()
    action = torch.randint(0, A, (B,), generator=g).cuda()
    return obs, cu.initial_inference(obs).latent_state, action


@pytest.mark.parametrize("B", [37, 300])
@pytest.mark.parametrize("name", NAMES)
def test_layers_match_float64(name, B):
    ref64, cu = make(name, "tc3")
    obs, latent, action = inputs(cu, name, B, 100 + B)
    for which, x0 in ((0, latent), (1, obs)):
        ratios, out, infos = run_program(cu, ref64, which, x0, action)
        print(f"\n[board-layers] {name} B={B} program {which}: " + " ".join(f"{k}={v:.3g}" for k, v in ratios.items()))
        bad = {k: r for k, r in ratios.items() if not r <= (0.25 if k.startswith("L") else 1.0)}
        assert not bad, f"{name} B={B} program {which}: over the bound {bad}"
        assert all(r > 0 for k, r in ratios.items() if k.endswith("head")), ratios   # an exact head is a dead one: bias only
        check_scalars(out, which, False, BR.BOARD_CONFIGS[name][6])
        nl = len(infos) - 1
        for L, info in enumerate(infos):
            assert info[4] == min(L + 1, nl) and info[5] == 3, info
            assert info[2] * info[0] >= B > (info[2] - 1) * info[0] and info[3] == B - (info[2] - 1) * info[0], info


@pytest.mark.parametrize("name", NAMES)
def test_bound_detects_single_pass(name):
    """tc1 (one fp16 pass) must exceed the bound by >= 8x on every 3x3 (wgmma) layer of both programs"""
    ref64, cu = make(name, "tc1")
    B = 37
    obs, latent, action = inputs(cu, name, B, 7)
    for which, x0 in ((0, latent), (1, obs)):
        ratios, _, infos = run_program(cu, ref64, which, x0, action)
        print(f"\n[board-layers tc1] {name} program {which}: " + " ".join(f"{k}={v:.3g}" for k, v in ratios.items()))
        assert all(info[5] == 1 for info in infos)
        weak = {k: r for k, r in ratios.items() if k.startswith("L") and not r >= 8.0}
        assert not weak, f"{name} program {which}: tc1 within 8x of the bound on {weak}"


# Every instantiation k_board_tc<C, NT> (C = 16, 32: NT = 1 .. 8; C = 64: NT = 1 .. 4) is its own straight-line code (its
# acc[NT][C / 2] accumulators, its fragment-row map, its ring waits): each runs both programs under the float64 check at a
# (board, B) whose launch plan has NT tiles.  NT -> (board, B): 1x1 boards pack up to 16 roots in one tile, so B = 1201 (10
# roots per CTA) stays at NT = 1; an 8x8 root takes 71 rows (NT = 2) and 132 of them fill one wave of one root each.
TILES = {1: ((1, 1), 1201), 2: ((8, 8), 132), 3: ((7, 8), 133), 4: ((7, 8), 265), 5: ((7, 8), 397), 6: ((7, 8), 529),
         7: ((8, 8), 529), 8: ((8, 8), 661)}
PAIRS = [(C, NT) for C in (16, 32, 64) for NT in range(1, (4 if C == 64 else 8) + 1)]


def tile_config(C, H, W):
    """a BOARD_CONFIGS-style config of C channels on an H x W board, one action per square"""
    return ((3, H, W), H * W, C, 1, 4, 16, (-10., 11., 1.))


@pytest.mark.parametrize("C,NT", PAIRS, ids=[f"C{C}_NT{NT}" for C, NT in PAIRS])
def test_every_tile_count_matches_float64(C, NT):
    """k_board_tc<C, NT> against float64 within the bounds of test_layers_match_float64 (tc3) and test_bound_detects_single_pass
    (tc1), and the public initial_inference / recurrent_inference outputs are the bits of the checked whole program"""
    (H, W), B = TILES[NT]
    cfg = tile_config(C, H, W)
    plan = BR.board_plan(C, H, W, B)
    assert plan[1] == NT, plan
    ref64, cu = make(cfg, "tc3")
    obs, latent, action = inputs(cu, cfg, B, 500 + NT)
    nres = cfg[3]
    for math in ("tc3", "tc1"):
        cu.set_math(math)
        for which, x0 in ((0, latent), (1, obs)):
            ratios, out, infos = run_program(cu, ref64, which, x0, action)
            print(f"\n[board-tiles] C={C} NT={NT} {H}x{W} B={B} plan={plan} {math} program {which}: "
                  + " ".join(f"{k}={v:.3g}" for k, v in ratios.items()))
            assert all(tuple(info[:4]) == plan and info[5] == (3 if math == "tc3" else 1) for info in infos), infos
            if math == "tc1":
                weak = {k: r for k, r in ratios.items() if k.startswith("L") and not r >= 8.0}
                assert not weak, f"C={C} NT={NT} program {which}: tc1 within 8x of the bound on {weak}"
                continue
            bad = {k: r for k, r in ratios.items() if not r <= (0.25 if k.startswith("L") else 1.0)}
            assert not bad, f"C={C} NT={NT} program {which}: over the bound {bad}"
            check_scalars(out, which, False, cfg[6])
            # the program the hook checked is the one the public entry points launch: the same bits
            lat, _ = board_stage(cu, which, x0, action, 2 * nres, len(infos) - 1)
            if which:
                o = cu.initial_inference(obs, return_scalar_value=True)
                pairs = [(o.latent_state, lat), (o.policy_logits, out["policy_logits"]), (o.value, out["value_logits"]),
                         (o.value_scalar, out["value"])]
            else:
                o = cu.recurrent_inference(latent, action.to(torch.int32), return_scalars=True)
                pairs = [(o.latent_state, lat), (o.policy_logits, out["policy_logits"]), (o.value, out["value_logits"]),
                         (o.reward, out["reward_logits"]), (o.value_scalar, out["value"]), (o.reward_scalar, out["reward"])]
            for i, (got, exp) in enumerate(pairs):
                assert torch.equal(got.reshape(-1), exp.reshape(-1)), (which, i)
