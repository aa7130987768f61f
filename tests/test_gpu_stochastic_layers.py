"""StochasticMuZeroModelMLP's tensor-core programs layer by layer against float64, and the bit identity a fused search relies on.

- Layers: the `init` (representation + prediction), `rec` (dynamics on afterstates + prediction) and `after` (afterstate
  dynamics + afterstate prediction, lz_model_debug_net_stage which = 2) programs, each layer on its own inputs (the kernel's
  output of the layer before), with the bounds of test_gpu_mlp_mz_layers.py: |y - y64| <= 2^-17 M + 2^-23 (M the magnitude sum
  of the layer) in tc3, and beyond it in tc1 on every layer and head -- a dropped hi / lo pass would fail.  The heads (hidden
  layer + FC2 pieces) are bounded through the magnitude of both Linears.  At L = 32 with A = C = K = 608 the `after` program is
  66 layers long, the kernel's limit.
- Bit identity: one root copied into every row gives the same bits at every row, in both recurrent programs, at NC = L / 32 of
  1, 2, 4 and 8; and under complementary row masks (the `after` program on some rows, `rec` on the others, as the search graph
  launches them) each selected row still has those bits, up to the partial last CTA, and no other row is written."""
import types

import pytest
import torch

import stoch_mlp_model_ref as SR
from test_gpu_mlp_ez_layers import layer_refs, linear
from test_gpu_mlp_mz_layers import head
from test_gpu_net_layers import worst

pytestmark = pytest.mark.gpu

TAU, ALPHA = 2.0 ** -17, 2.0 ** -23
B = 129
NAMES = list(SR.CONFIGS)


def make(name, math="tc3"):
    import lightzero_b200 as lzb
    ref = SR.build(name, NAMES.index(name))
    cu = lzb.StochasticMuZeroModelMLP(**SR.model_kwargs(name)).load_state_dict(ref.state_dict())
    cu.set_math(math)
    return ref, cu


def program_ref(ref, which):
    """the networks of a program under the names layer_refs reads: which 1 init, 0 rec, 2 after"""
    if which == 2:
        return types.SimpleNamespace(representation_network=ref.representation_network,
                                     dynamics_network=ref.afterstate_dynamics_network,
                                     prediction_network=ref.afterstate_prediction_network)
    return ref


def stage(cu, which, x, option, s):
    from lightzero_b200 import cabi
    L, K = cu.latent_state_dim, cu.value_support_size
    P = cu.chance_space_size if which == 2 else cu.action_space_size
    n = x.shape[0]
    out = torch.zeros(n * (2 * K + P + 2 + 2 * L), device="cuda")
    info = (cabi.ctypes.c_int32 * 8)()
    cabi.check(cu._lib.lz_model_debug_net_stage(cu._h, which, n, x.contiguous().data_ptr(), option.data_ptr(), s, out.data_ptr(),
                                                out.numel() * 4, info, cabi.stream_ptr()), "lz_model_debug_net_stage")
    torch.cuda.synchronize()
    D = info[7]
    if s < D:
        return out[:n * L].view(n, L).double().cpu(), list(info)
    v = out.cpu().double()[2 * n * L:]
    o = dict(value=v[:n * K].view(n, K), policy=v[n * K:n * (K + P)].view(n, P))
    if which != 1:
        o["reward"] = v[n * (K + P + 1):n * (2 * K + P + 1)].view(n, K)
    return o, list(info)


def program_inputs(cu, which, seed=77):
    """(x0 float64 [B, in], option int32 [B] on the device, one-hot width): observations for init, latents and actions for
    after, the kernel's own afterstates and chance outcomes for rec"""
    A, C = cu.action_space_size, cu.chance_space_size
    g = torch.Generator().manual_seed(seed)
    obs = torch.rand((B, cu.observation_shape), generator=g) * 2.0 - 1.0
    act, ch = torch.randint(0, A, (B,), generator=g), torch.randint(0, C, (B,), generator=g)
    if which == 1:
        return obs.double(), act.int().cuda(), A
    lat = cu.initial_inference(obs.cuda()).latent_state
    if which == 2:
        return lat.double().cpu(), act.int().cuda(), A
    after = cu.recurrent_inference(lat, act.cuda(), afterstate=False).latent_state
    return after.double().cpu(), ch.int().cuda(), C


def ratios(name, ref, cu, which):
    """{layer: worst |err| / bound} of one program, and the launch info of the whole program"""
    res = SR.CONFIGS[name][4]
    x0, option, n1 = program_inputs(cu, which)
    onehot = torch.nn.functional.one_hot(option.long().cpu(), n1).double()
    net = program_ref(ref, which)
    layers = layer_refs(net, 1 if which == 1 else 0)
    D = len(layers)
    prev, z, dumps, r = x0, x0, [], {}
    for s, (lin, bn, act, oh, resid, ln) in enumerate(layers):
        got, info = stage(cu, which, x0.float().cuda(), option, s)
        assert info[7] == D
        if res and which != 1 and s == 4:
            prev = dumps[1]             # the prediction reads next = fc_dynamics_1 + state, not fc_dynamics_2's output
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
    whole, info = stage(cu, which, x0.float().cuda(), option, D)
    P = net.prediction_network
    heads = [("value", P.fc_value_head, prev), ("policy", P.fc_policy_head, prev)]
    if which != 1:
        heads.append(("reward", net.dynamics_network.fc_reward_head, dumps[3] if res else dumps[1]))
    for key, mlp, x in heads:
        y, M = head(mlp, x)
        r[key] = worst(whole[key] - y, TAU * M + ALPHA)
    return r, info


PROGRAMS = {"init": 1, "rec": 0, "after": 2}


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("program", list(PROGRAMS))
def test_layers_match_float64_and_tc1_fails(name, program):
    which = PROGRAMS[program]
    ref, cu = make(name)
    r3, info = ratios(name, ref, cu, which)
    print(f"\n[stochastic-layers] {name} NC={cu.latent_state_dim // 32} {program} layers={info[3]} tc3 "
          + " ".join(f"{k}={v:.3g}" for k, v in r3.items()))
    assert all(v <= 1.0 for v in r3.values()), r3
    assert which == 1 or "reward" in r3
    if name == "l32_a608_c608" and which != 1:
        assert info[3] == 66            # the longest program the kernel takes (kMezMaxLayers)
    # a head whose hidden units are all inactive on these inputs (one unit at l32_c1_h1) is its FC2 bias, exact in any mode
    exact = {k for k, v in r3.items() if v == 0.0}
    assert exact <= {"value", "reward", "policy"} and len(exact) <= 1, exact
    cu.set_math("tc1")                  # a math mode: the tensor-core kernel, not the fp32 one
    r1, _ = ratios(name, ref, cu, which)
    print(f"[stochastic-layers] {name} {program} tc1 " + " ".join(f"{k}={v:.3g}" for k, v in r1.items()))
    assert all(v > 1.0 for k, v in r1.items() if k not in exact) and all(r1[k] == 0.0 for k in exact), r1


def test_after_stage_refused_by_other_models():
    """which 2 is the afterstate program: a MuZeroModelMLP on the same kernel refuses it"""
    from lightzero_b200 import cabi
    from test_gpu_mlp_mz import make as make_mz
    _, mz = make_mz("lunarlander")
    x = torch.zeros(4, 256, device="cuda")
    a = torch.zeros(4, dtype=torch.int32, device="cuda")
    out = torch.zeros(4 * 2000, device="cuda")
    info = (cabi.ctypes.c_int32 * 8)()
    with pytest.raises(cabi.LzError, match="afterstate"):
        cabi.check(mz._lib.lz_model_debug_net_stage(mz._h, 2, 4, x.data_ptr(), a.data_ptr(), 0, out.data_ptr(), out.numel() * 4,
                                                    info, cabi.stream_ptr()), "lz_model_debug_net_stage")


def _outs(cu, n, P):
    shapes = ((n, cu.latent_state_dim), (n, cu.reward_support_size), (n, cu.value_support_size), (n, P), (n,), (n,))
    return [torch.full(s, 7.25, device="cuda") for s in shapes]


@pytest.mark.parametrize("name", ["l32_c1_h1", "l64_c9_res", "cartpole", "lunarlander_disc"])
def test_one_root_same_bits_at_every_row(name):
    """NC = L / 32 of 1, 2, 4, 8: a root copied into all rows of 2 CTAs and a partial third gives the bits of the root alone at
    every row, in the `after` and `rec` programs; with complementary row masks over the same state and option buffers (after
    on the rows whose bit is set, rec on the others) every selected row keeps those bits and every other row is untouched"""
    from lightzero_b200 import cabi
    _, cu = make(name)
    A, C, L = cu.action_space_size, cu.chance_space_size, cu.latent_state_dim
    n = 2 * 64 + 37
    g = torch.Generator().manual_seed(5)
    lat = cu.initial_inference((torch.rand((1, cu.observation_shape), generator=g) * 2 - 1).cuda()).latent_state
    a0 = torch.tensor([A - 1], dtype=torch.int32, device="cuda")
    c0 = torch.tensor([C - 1], dtype=torch.int32, device="cuda")
    aft = cu.recurrent_inference(lat, a0, afterstate=False).latent_state
    one = {False: cu.recurrent_inference(lat, a0, False, return_scalars=True),
           True: cu.recurrent_inference(aft, c0, True, return_scalars=True)}
    fields = ("latent_state", "reward", "value", "policy_logits", "reward_scalar", "value_scalar")
    for afterstate, (x, o) in ((False, (lat, a0)), (True, (aft, c0))):
        many = cu.recurrent_inference(x.repeat(n, 1), o.repeat(n), afterstate, return_scalars=True)
        for f in fields:
            assert torch.equal(getattr(many, f), getattr(one[afterstate], f).expand_as(getattr(many, f))), (afterstate, f)
    mask = (torch.rand(n, generator=g) < 0.5).int().cuda()
    mask[64:128] = 1                                    # a CTA the rec launch skips ...
    mask[128:] = 0                                      # ... and a partial last CTA the after launch skips
    sel = mask.bool()
    state = torch.where(sel[:, None], lat.expand(n, L), aft.expand(n, L)).contiguous()
    opt = torch.where(sel, a0.expand(n), c0.expand(n)).contiguous()
    for afterstate, on in ((False, 1), (True, 0)):
        outs = _outs(cu, n, A if afterstate else C)
        cabi.check(cu._lib.lz_model_recurrent_inference_stochastic(cu._h, int(afterstate), n, state.data_ptr(), opt.data_ptr(),
                                                               mask.data_ptr(), on, *(t.data_ptr() for t in outs),
                                                               cabi.stream_ptr()), "masked")
        rows = sel if on else ~sel
        for f, got in zip(fields, outs):
            e = getattr(one[afterstate], f)
            assert torch.equal(got[rows], e.expand((int(rows.sum()),) + tuple(e.shape[1:]))), (afterstate, f)
            assert bool((got[~rows] == 7.25).all()), (afterstate, f)
