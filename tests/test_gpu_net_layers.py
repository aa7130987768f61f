"""The latent-grid tensor-core network (k_net_tc) layer by layer against float64 (lz_model_debug_net_stage).

The hook runs a copy of the recurrent program (dynamics conv, dynamics ResBlocks, prediction ResBlocks, heads) or of the
initial_inference tail (representation ResBlocks, prediction ResBlocks, value / policy heads) cut off after one layer,
and returns that layer's fp32 output.  Each layer's reference runs in float64 on exactly the operands the kernel
consumed: the previous dump split the way the kernel splits it (hi = fp16(min(v, 65504)), lo = fp16(v - hi)) as the
MMA input, and the unsplit fp32 dump as the ResBlock residual (the skip scratch holds fp32).  A layer's error is then its
own, and it is compared element by element with

    |y_cuda - y_f64| <= TAU[kind] * M + ALPHA * S

M is the layer evaluated in float64 on |W|, |x|, the BatchNorm terms |scale| (|conv| + |mean|) + |beta| and |residual|;
S counts the operands whose fp16 lo part can be subnormal (2^-25 absolute each).  Layer 0 is conv(latent | one-hot)
-> BN -> + latent -> ReLU; the kernel adds the one-hot part as a precomputed fp32 table, whose rounding TAU covers.

Each head is one stage: 1x1 conv -> BN -> ReLU -> FC1 -> BN1d -> ReLU -> FC2 on the split output of the layer it hooks,
with M and S carried through the chain.  The scalars are h^-1 of the softmax expectation of the kernel's own logits
(DESIGN.md 4.4), and must be bit-identical whether the raw logits are requested or not (the joint read-out).

TAU is calibrated on an H100 (DESIGN.md 4.3) so that 3xFP16 stays under a quarter of the bound; a single fp16 pass
(tc1) exceeds it by >= 8x on every 3x3 layer and on each head's 1x1 conv.  FC1 and FC2 always issue both A parts, so
for them the same margin is shown in float64: dropping the weights' lo parts in the reference must exceed the bound.
"""
import copy

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

N_SMS = 132
ALPHA = 2.0 ** -23
# calibrated per layer kind (DESIGN.md 4.3); a head's M sums |W2| |W1| |features| without cancellation, hence its small TAU
TAU = {"dyn": 2.0 ** -17, "conv1": 2.0 ** -17, "conv2": 2.0 ** -17, "value": 2.0 ** -23, "reward": 2.0 ** -23,
       "policy": 1e-7, "feat": 2.0 ** -17, "lstm": 2.0 ** -17}
SUPPORT = (-300., 301., 1.)
EXPF_ERR = 2e-6          # the __expf / __fdividef sigmoid and tanh of the LSTM cell (DESIGN.md 4.5: ~1e-6)


# ------------------------------------------------------------------------------------------------ models and inputs
def make_models(A=6, nres=1, hc=(16, 16, 16), hid=32, support=SUPPORT, seed=0, math="tc3", ez=False, mutate=None):
    """(float64 reference on the GPU, CUDA model); hc = (reward, value, policy) head channels"""
    import lightzero_b200 as lzb
    from oracle.model_ref import EfficientZeroModelRef, MuZeroModelRef, emulate_trained_
    torch.manual_seed(seed)
    kw = dict(num_res_blocks=nres, reward_head_channels=hc[0], value_head_channels=hc[1], policy_head_channels=hc[2],
              reward_head_hidden_channels=(hid,), value_head_hidden_channels=(hid,), policy_head_hidden_channels=(hid,),
              reward_support_range=support, value_support_range=support)
    obs = (4, 96, 96) if ez else (4, 84, 84)
    ref = emulate_trained_((EfficientZeroModelRef if ez else MuZeroModelRef)(obs, A, **kw), seed)
    if mutate is not None:
        mutate(ref)
    cu = (lzb.EfficientZeroModel if ez else lzb.MuZeroModel)(observation_shape=obs, action_space_size=A, **kw)
    cu.load_state_dict(ref.state_dict())
    cu.set_math(math)
    return copy.deepcopy(ref).double().cuda().eval(), cu


SCALES = (0.0, 1e-3, 0.05, 1.0, 1.0, 4.0, 30.0, 2e3)


def make_latents(B, seed, peak=None):
    """post-ReLU latents with a per-root scale: all-zero roots, roots whose lo parts are fp16-subnormal, unit roots
    and large ones; `peak` rescales the largest class so that the batch maximum is `peak`"""
    g = torch.Generator().manual_seed(seed)
    x = torch.relu(torch.randn(B, 64, 6, 6, generator=g))
    s = torch.tensor(SCALES, dtype=torch.float32)[torch.randint(0, len(SCALES), (B,), generator=g)]
    x = x * s.view(-1, 1, 1, 1)
    if peak is not None and x.max() > 0:
        x = x * (peak / x.max())
    return x.cuda()


def pick_roots(B):
    """tc_pick_roots: at most one wave of one CTA per SM, at most 8 roots per CTA"""
    return min(max(-(-B // N_SMS), 1), 8)


# ------------------------------------------------------------------------------------------------ the hook
def net_stage(cu, which, latent, action, stage, nlayers):
    """(f32 output, h_info) of the program cut after layer `stage` (stage == nlayers: the whole program)"""
    from lightzero_b200 import cabi
    B, K, A = latent.shape[0], cu.value_support_size, cu.action_space_size
    nfeat = cu._cfg.reward_head_channels * 36 if cu._cfg.efficientzero else 0
    n = B * 2304 if stage < nlayers else B * (2 * K + 2 * A + 4 + nfeat)
    buf = torch.full((n,), float("nan"), dtype=torch.float32, device="cuda")
    info = np.zeros(8, np.int32)
    act = action.to(torch.int32).contiguous() if action is not None else None
    cabi.check(cu._lib.lz_model_debug_net_stage(cu._h, which, B, latent.contiguous().data_ptr(), cabi.ptr(act), stage,
                                                buf.data_ptr(), buf.numel() * 4, info.ctypes.data, cabi.stream_ptr()),
               "lz_model_debug_net_stage")
    torch.cuda.synchronize()
    return buf, [int(v) for v in info]


def split_full(buf, B, K, A, nfeat):
    sizes = [B * K, B * K, B * A, B, B, B * A, B, B, B * nfeat]
    rl, vl, pl, r, v, pl2, r2, v2, feat = torch.split(buf, sizes)
    return dict(reward_logits=rl.view(B, K), value_logits=vl.view(B, K), policy_logits=pl.view(B, A), reward=r, value=v,
                policy_logits2=pl2.view(B, A), reward2=r2, value2=v2, feat=feat.view(B, nfeat))


# ------------------------------------------------------------------------------------------------ float64 references
def split_hi_lo(v):
    """float64 value of the kernel's fp16 hi/lo split of an fp32 activation (store_split8 / store_split8_pos: the
    value is clamped to the fp16 range first)"""
    a = v.float().clamp(-65504.0, 65504.0)
    hi = a.half()
    return hi.double() + (a - hi.float()).half().double()


def _bn(bn, shape):
    s = bn.weight / torch.sqrt(bn.running_var + bn.eps)
    return s.view(shape), bn.running_mean.view(shape), bn.bias.view(shape)


def program(ref64, which):
    """[(conv, bn, kind)] of the recurrent (0) or tail (1) program, and the layer the reward head hooks"""
    dyn, pred, rep = ref64.dynamics_network, ref64.prediction_network, ref64.representation_network
    layers, blocks = [], list(pred.resblocks)
    if which == 0:
        layers.append((dyn.conv, dyn.norm_common, "dyn"))
        blocks = list(dyn.resblocks) + blocks
    else:
        blocks = list(rep.resblocks) + blocks
    for b in blocks:
        layers += [(b.conv1[0], b.conv1[1], "conv1"), (b.conv2[0], b.conv2[1], "conv2")]
    return layers, (2 * len(dyn.resblocks) if which == 0 else None)


def layer_reference(conv, bn, kind, x, res, onehot):
    """(y, M, S) of one 3x3 layer on the split input x (+ the fp32 residual res)"""
    W = conv.weight
    xin, Min = (torch.cat([x, onehot], 1), torch.cat([x.abs(), onehot], 1)) if kind == "dyn" else (x, x.abs())
    y, M = F.conv2d(xin, W, padding=1), F.conv2d(Min, W.abs(), padding=1)
    s, mean, beta = _bn(bn, (1, -1, 1, 1))
    y, M = s * (y - mean) + beta, s.abs() * (M + mean.abs()) + beta.abs()
    if res is not None:
        y, M = y + res, M + res.abs()
    return torch.relu(y), M, torch.ones_like(M)


def pow2_hi(w):
    """the fp16 hi part of a weight matrix as the host packs it: scaled by a power of two so that max |w| lands in
    [4096, 8192), rounded to fp16, scaled back"""
    _, e = torch.frexp(w.abs().max())
    scale = 2.0 ** (13 - int(e))
    return (w * scale).float().half().double() / scale


def head_features(conv, bn, x):
    """1x1 conv -> BN -> ReLU on the split hook output x: (features, M) flattened as [B][c * 36 + p]"""
    z, Mz = F.conv2d(x, conv.weight, conv.bias), F.conv2d(x.abs(), conv.weight.abs(), conv.bias.abs())
    s, mean, beta = _bn(bn, (1, -1, 1, 1))
    return torch.relu(s * (z - mean) + beta).flatten(1), (s.abs() * (Mz + mean.abs()) + beta.abs()).flatten(1)


def head_reference(conv, bn, mlp, x, hi_only=False):
    """(logits, M, S) of one head on the split hook output x; hi_only drops the FC weights' lo parts"""
    f, Mf = head_features(conv, bn, x)
    lin1, bn1, lin2 = mlp[0], mlp[1], mlp[3]
    W1, W2 = (pow2_hi(lin1.weight), pow2_hi(lin2.weight)) if hi_only else (lin1.weight, lin2.weight)
    s1, m1, b1 = _bn(bn1, (1, -1))
    u, Mu = f @ W1.T + lin1.bias, Mf @ W1.abs().T + lin1.bias.abs()
    g, Mg = torch.relu(s1 * (u - m1) + b1), s1.abs() * (Mu + m1.abs()) + b1.abs()
    Sg = s1.abs() * (torch.ones_like(f) @ W1.abs().T) + 1.0
    return g @ W2.T + lin2.bias, Mg @ W2.abs().T + lin2.bias.abs(), Sg @ W2.abs().T + 1.0


def inverse_h(logits, support):
    """h^-1 of the softmax expectation, float64 (scaling_transform.py:64-92)"""
    sup = torch.arange(*support, dtype=torch.float64, device=logits.device)
    v = (torch.softmax(logits.double(), 1) * sup).sum(1)
    eps = 0.001
    t = (torch.sqrt(1 + 4 * eps * (v.abs() + 1 + eps)) - 1) / (2 * eps)
    return torch.sign(v) * (t * t - 1)


def worst(err, bound):
    return (err.abs() / bound).max().item() if err.numel() else 0.0


def run_program(cu, ref64, which, latent, action, support=SUPPORT, hi_only=False):
    """Every layer and head of one program against float64.  Returns (ratios {stage: worst |err| / bound}, dumps,
    full outputs, infos); ratios of the heads with hi_only are those of the hi-only float64 reference instead"""
    layers, rew_hook = program(ref64, which)
    nl, B, A = len(layers), latent.shape[0], cu.action_space_size
    ez = bool(cu._cfg.efficientzero)
    dumps, infos = [], []
    for L in range(nl):
        buf, info = net_stage(cu, which, latent, action, L, nl)
        dumps.append(buf.view(B, 64, 6, 6).double())
        infos.append(info)
    buf, info = net_stage(cu, which, latent, action, nl, nl)
    infos.append(info)
    out = split_full(buf, B, cu.value_support_size, A, cu._cfg.reward_head_channels * 36 if ez else 0)
    x0 = latent.double()
    onehot = None
    if which == 0:
        onehot = F.one_hot(action.long(), A).double().view(B, A, 1, 1).expand(B, A, 6, 6)
    ratios = {}
    with torch.no_grad():
        for L, (conv, bn, kind) in enumerate(layers):
            res = None
            if kind == "dyn":
                res = x0
            elif kind == "conv2":
                res = dumps[L - 2] if L >= 2 else x0
            y, M, S = layer_reference(conv, bn, kind, split_hi_lo(dumps[L - 1] if L else x0), res, onehot)
            ratios[f"L{L}:{kind}"] = worst(dumps[L] - y, TAU[kind] * M + ALPHA * S)
        pred, dyn = ref64.prediction_network, ref64.dynamics_network
        xl = split_hi_lo(dumps[nl - 1])
        heads = [("value", pred.conv1x1_value, pred.norm_value, pred.fc_value, xl, out["value_logits"]),
                 ("policy", pred.conv1x1_policy, pred.norm_policy, pred.fc_policy, xl, out["policy_logits"])]
        if which == 0 and not ez:
            heads.append(("reward", dyn.conv1x1_reward, dyn.norm_reward, dyn.fc_reward_head, split_hi_lo(dumps[rew_hook]),
                          out["reward_logits"]))
        for name, conv, bn, mlp, x, got in heads:
            y, M, S = head_reference(conv, bn, mlp, x)
            bound = TAU[name] * M + ALPHA * S
            if hi_only:
                ratios[f"{name} head"] = worst(head_reference(conv, bn, mlp, x, hi_only=True)[0] - y, bound)
            else:
                ratios[f"{name} head"] = worst(got.double() - y, bound)
        if which == 0 and ez:
            f, Mf = head_features(dyn.conv1x1_reward, dyn.norm_reward, split_hi_lo(dumps[rew_hook]))
            ratios["ez_feat"] = worst(out["feat"].double() - f, TAU["feat"] * Mf + ALPHA)
    return ratios, dumps, out, infos


def check_scalars(out, which, ez, support=SUPPORT):
    """the scalars against h^-1 of the kernel's own logits, and bit identity with the joint read-out"""
    for name in (("value", "reward") if which == 0 and not ez else ("value",)):
        got, exp = out[name].double(), inverse_h(out[f"{name}_logits"], support)
        assert torch.isfinite(got).all(), name
        bad = (got - exp).abs() > 2e-4 * torch.clamp(exp.abs(), min=1.0)
        assert not bad.any(), (name, int(bad.sum()), (got - exp).abs().max().item())
        assert torch.equal(out[name], out[f"{name}2"]), f"{name}: the joint categorical read-out differs"
    assert torch.equal(out["policy_logits"], out["policy_logits2"])


def check_plan(info, B, nlayers, npass):
    """h_info: R, NT, CTAs, roots of the last CTA, layers launched, passes"""
    R = pick_roots(B)
    ctas = -(-B // R)
    assert info[:6] == [R, (49 * R - 8 + 127) >> 7, ctas, B - (ctas - 1) * R, nlayers, npass], (B, info)


# ------------------------------------------------------------------------------------------------ CTA packings
PACK_B = (1, 131, 133, 265, 395, 397, 531, 667, 799, 1023, 1024, 1201)
_DEFAULT = {}


def _default(math="tc3"):
    if math not in _DEFAULT:
        _DEFAULT[math] = make_models(A=18, seed=11, math=math)
    return _DEFAULT[math]


@pytest.mark.parametrize("which", [0, 1])
@pytest.mark.parametrize("B", PACK_B)
def test_packing_matches_float64(B, which):
    ref64, cu = _default()
    latent = make_latents(B, seed=B)
    action = (torch.arange(B) % cu.action_space_size).cuda()
    ratios, _, out, infos = run_program(cu, ref64, which, latent, action)
    bad = {k: r for k, r in ratios.items() if not r <= 1.0}
    assert not bad, f"B = {B}: over the float64 bound (worst |err| / bound): {bad}"
    check_scalars(out, which, False)
    nl = len(infos) - 1
    for L, info in enumerate(infos):
        check_plan(info, B, min(L + 1, nl), 3)


def test_packings_cover_every_cta_shape():
    """R = 1 .. 8, a last CTA of one root for R = 2 .. 8, a partial last CTA of several roots and a second wave"""
    plans = {B: (pick_roots(B), -(-B // pick_roots(B))) for B in PACK_B}
    last = {B: B - (c - 1) * R for B, (R, c) in plans.items()}
    assert {R for R, _ in plans.values()} == set(range(1, 9))
    assert all(any(R == r and last[B] == 1 for B, (R, _) in plans.items()) for r in range(2, 9))
    assert any(1 < last[B] < R for B, (R, _) in plans.items())
    assert any(c > N_SMS for _, c in plans.values())


# ------------------------------------------------------------------------------------------------ configurations
# (A, num_res_blocks, head channels (reward, value, policy), head hidden, support): every value of each dimension
CONFIGS = [
    (6, 1, (16, 16, 16), 32, SUPPORT),
    (334, 1, (8, 1, 16), 32, SUPPORT),          # the last A whose FC2 biases are staged in shared memory (nres = 1, K = 601)
    (335, 1, (16, 8, 1), 8, SUPPORT),           # the first that reads them from global memory
    (608, 2, (1, 16, 8), 8, (-304., 304., 1.)),   # the largest heads: K = A = 608, 3 x 5 = 15 FC2 tiles
    (1, 3, (8, 8, 8), 32, (-10., 11., 1.)),
    (32, 4, (16, 1, 8), 8, (-10., 11., 1.)),    # 17 layers, the longest program
    (33, 2, (1, 1, 1), 32, (-304., 304., 1.)),
    (129, 1, (8, 16, 8), 8, (-10., 11., 1.)),
    (608, 1, (16, 8, 1), 32, (-10., 11., 1.)),    # staged biases with 5 policy tiles
]


def _cfg_id(c):
    A, n, hc, hid, sup = c
    return f"A{A}-nres{n}-hc{'.'.join(map(str, hc))}-hid{hid}-K{len(np.arange(*sup))}"


@pytest.mark.parametrize("cfg", CONFIGS, ids=[_cfg_id(c) for c in CONFIGS])
def test_configuration_matches_float64(cfg):
    A, nres, hc, hid, support = cfg
    ref64, cu = make_models(A=A, nres=nres, hc=hc, hid=hid, support=support, seed=A + nres)
    for which, B in ((0, 397), (0, 131), (1, 397)):
        latent = make_latents(B, seed=A + B)
        action = (torch.arange(B) % A).cuda()
        ratios, _, out, infos = run_program(cu, ref64, which, latent, action, support)
        bad = {k: r for k, r in ratios.items() if not r <= 1.0}
        assert not bad, f"{_cfg_id(cfg)} which={which} B={B}: over the float64 bound: {bad}"
        check_scalars(out, which, False, support)
        if which == 0:
            K = len(np.arange(*support))
            assert infos[-1][7] == 2 * (-(-K // 128)) + (-(-A // 128)), infos[-1]
            assert infos[-1][6] == int((infos[-1][4] * 128 + 2 * K + A) <= 2176), infos[-1]


def test_configurations_cover_every_value():
    assert {c[0] for c in CONFIGS} >= {1, 6, 32, 33, 129, 334, 335, 608}
    assert {c[1] for c in CONFIGS} == {1, 2, 3, 4}
    assert {h for c in CONFIGS for h in c[2]} == {16, 8, 1}
    assert {c[3] for c in CONFIGS} == {32, 8}
    assert {len(np.arange(*c[4])) for c in CONFIGS} == {601, 21, 608}
    # both sides of the FC2-bias staging threshold of the recurrent program (5 layers at nres = 1)
    staged = {c[0]: (5 * 128 + 2 * len(np.arange(*c[4])) + c[0]) <= 2176 for c in CONFIGS if c[1] == 1}
    assert staged[334] and not staged[335]


def test_heads_over_608_outputs_are_refused():
    """The FC2 staging of k_net_tc holds heads of up to 608 outputs: a larger action space is refused at finalize."""
    from lightzero_b200.cabi import LzError
    with pytest.raises(LzError, match="608"):
        make_models(A=609)


# ------------------------------------------------------------------------------------------------ bit identity
def _slot_batches(T, Ta, B, A, seed):
    """a batch of B roots in which test root t sits at slots 0 .. R-1 of CTA t"""
    R = pick_roots(B)
    latent = make_latents(B, seed)
    action = (torch.arange(B) % A).cuda()
    pos = {}
    for t in range(T.shape[0]):
        for s in range(R):
            p = t * R + s
            latent[p], action[p] = T[t], Ta[t]
            pos.setdefault(t, []).append(p)
    return latent, action, pos


def _outputs(cu, which, latent, action, nl):
    """(last layer dump, full outputs) of one program"""
    last, _ = net_stage(cu, which, latent, action, nl - 1, nl)
    full, _ = net_stage(cu, which, latent, action, nl, nl)
    B = latent.shape[0]
    out = split_full(full, B, cu.value_support_size, cu.action_space_size, 0)
    return last.view(B, -1), out


@pytest.mark.parametrize("hc", [16, 8])
def test_root_outputs_identical_at_every_slot_and_packing(hc):
    """A root's outputs are the same bits at every slot of a CTA, at every R, on repeated calls and with the workspace
    reused: rows of one root never mix with another's, and every row sums in one fixed order."""
    A = 6
    ref64, cu = make_models(A=A, hc=(hc, hc, hc), seed=5)
    T = make_latents(8, seed=99)
    T[0] = 0.0                                            # an all-zero root
    T[1] = T[1] * (1e-3 / max(T[1].max().item(), 1e-30))  # lo parts in the fp16 subnormal range
    Ta = (torch.arange(8) % A).cuda()
    for which in (0, 1):
        nl = len(program(ref64, which)[0])
        alone = [_outputs(cu, which, T[t:t + 1].contiguous(), Ta[t:t + 1].contiguous(), nl) for t in range(8)]
        for B in (131, 133, 265, 397, 531, 667, 799, 1023, 1201, 131):
            latent, action, pos = _slot_batches(T, Ta, B, A, seed=B + which)
            for rep in range(2 if B == 1023 else 1):
                last, out = _outputs(cu, which, latent, action, nl)
                for t, ps in pos.items():
                    a_last, a_out = alone[t]
                    for p in ps:
                        assert torch.equal(last[p], a_last[0]), (which, B, t, p)
                        for k in ("value_logits", "policy_logits", "value", "policy_logits2", "value2") + (
                                ("reward_logits", "reward", "reward2") if which == 0 else ()):
                            assert torch.equal(out[k][p], a_out[k][0]), (which, B, t, p, k)


# ------------------------------------------------------------------------------------------------ sensitivity
def test_bound_detects_single_pass():
    """tc1 (one fp16 pass) must exceed the bound by >= 8x on every 3x3 layer and on every head (its 1x1 conv)."""
    ref64, cu = _default("tc1")
    B = 397
    latent, action = make_latents(B, seed=3), (torch.arange(B) % cu.action_space_size).cuda()
    for which in (0, 1):
        ratios, _, _, infos = run_program(cu, ref64, which, latent, action)
        assert all(info[5] == 1 for info in infos)
        weak = {k: r for k, r in ratios.items() if not r >= 8.0}
        assert not weak, f"which={which}: tc1 within 8x of the bound: {weak}"


def test_head_bound_detects_dropped_weight_lo_parts():
    """FC1 / FC2 always issue A_hi and A_lo; the float64 head reference with the weights' lo parts dropped must exceed
    the head bound by >= 8x, so a lost FC pass would be seen."""
    ref64, cu = _default()
    B = 397
    latent, action = make_latents(B, seed=4), (torch.arange(B) % cu.action_space_size).cuda()
    ratios, _, _, _ = run_program(cu, ref64, 0, latent, action, hi_only=True)
    weak = {k: r for k, r in ratios.items() if k.endswith("head") and not r >= 8.0}
    assert not weak, weak


# ------------------------------------------------------------------------------------------------ wide range
def _wide_range(ref):
    """per-output-channel conv weight multipliers 2^-8 .. 2^2 on the latent-grid convs and BatchNorm variances down to
    1e-3 on the small channels"""
    g = torch.Generator().manual_seed(17)
    with torch.no_grad():
        for net in (ref.dynamics_network, ref.prediction_network, ref.representation_network):
            for blk in net.resblocks:
                for seq in (blk.conv1, blk.conv2):
                    co = seq[0].weight.shape[0]
                    e = torch.linspace(-8.0, 2.0, co)[torch.randperm(co, generator=g)]
                    seq[0].weight.mul_((2.0 ** e).view(-1, 1, 1, 1))
                    small = e <= -3
                    seq[1].running_var[small] = 1e-3 * (1.0 + torch.rand(int(small.sum()), generator=g))


def test_wide_range_model():
    """Channels whose weights are 2^-8 of the largest leave subnormal lo parts after the power-of-two weight scale;
    large inputs push activations towards the fp16 maximum (~6e4)."""
    ref64, cu = make_models(A=18, seed=23, mutate=_wide_range)
    B = 531
    latent, action = make_latents(B, seed=8, peak=3.5e4), (torch.arange(B) % 18).cuda()
    for which in (0, 1):
        ratios, dumps, out, _ = run_program(cu, ref64, which, latent, action)
        assert max(d.abs().max().item() for d in dumps) > 3e4
        assert max(ratios.values()) <= 1.0, ratios
        check_scalars(out, which, False)


# ------------------------------------------------------------------------------------------------ persistent search
class _Recorder:
    """Wraps the CUDA model so the step-wise search records what the network returned."""

    def __init__(self, model):
        self.model, self.calls = model, []

    def eval(self):
        return self

    def recurrent_inference(self, latent, action):
        out = self.model.recurrent_inference(latent, action, return_scalars=True)
        self.calls.append((latent.clone(), action.clone(), out))
        return out


@pytest.mark.parametrize("B", [131, 531, 799])
def test_persistent_search_with_narrow_heads(B):
    """Head channels 8 (FC1 inputs 288 of 576) in the persistent search kernel: fused == step-wise drive bit for bit,
    every root value finite, and every network call of the step-wise drive within the float64 replay's tolerance."""
    import lightzero_b200 as lzb
    from oracle.model_ref import DiscreteSupport, InverseScalarTransform
    A, S = 6, 20
    ref64, cu = make_models(A=A, hc=(8, 8, 8), seed=B)
    rng = np.random.default_rng(B)
    obs = torch.rand(B, 4, 84, 84, generator=torch.Generator().manual_seed(B)).cuda()
    out = cu.initial_inference(obs)
    legal = [list(range(A))] * B
    noises = [rng.dirichlet([0.3] * A).astype(np.float32).tolist() for _ in range(B)]
    mcts = lzb.MuZeroMCTSCtree(dict(num_simulations=S, deterministic=True, discount_factor=0.997))
    results, rec = [], _Recorder(cu)
    for mode in ("fused", "step"):
        roots = mcts.roots(B, legal)
        roots.prepare(0.25, noises, [0.] * B, out.policy_logits, [-1] * B)
        mcts.search(roots, cu if mode == "fused" else rec, out.latent_state, [-1] * B)
        if mode == "fused":
            assert mcts.last_num_kernels == 1
        vals = np.asarray(roots.get_values(), np.float32)
        assert np.isfinite(vals).all()
        results.append((roots.get_distributions(), vals.view(np.uint32).tolist()))
        roots.clear()
    assert results[0] == results[1]
    inv = InverseScalarTransform(DiscreteSupport(*SUPPORT))
    for latent, action, o in rec.calls:
        with torch.no_grad():
            exp = ref64.recurrent_inference(latent.double(), action.reshape(-1).long())
        for a, e in ((o.latent_state, exp.latent_state), (o.reward, exp.reward), (o.value, exp.value),
                     (o.policy_logits, exp.policy_logits)):
            assert torch.allclose(a.double(), e, rtol=1e-5, atol=1e-5), (a.double() - e).abs().max().item()
        with torch.no_grad():
            ev, er = inv(exp.value.float().cpu()).reshape(-1), inv(exp.reward.float().cpu()).reshape(-1)
        assert torch.allclose(o.value_scalar.cpu(), ev, rtol=2e-4, atol=2e-4)
        assert torch.allclose(o.reward_scalar.cpu(), er, rtol=2e-4, atol=2e-4)


# ------------------------------------------------------------------------------------------------ EfficientZero
def lstm_bound(lstm, feat, h0, c0, tau=TAU["lstm"], weights=None):
    """float64 (h1, c1) of one nn.LSTM step and their error bounds: tau * M on the gate pre-activations, carried through
    sigmoid / tanh (Lipschitz 1/4 and 1), plus the error of the fast sigmoid / tanh.  `weights`: (W_ih, W_hh) to use
    instead of the module's (the bound is always taken on the module's)"""
    Wi, Wh, b = lstm.weight_ih_l0, lstm.weight_hh_l0, lstm.bias_ih_l0 + lstm.bias_hh_l0
    z = feat @ (weights[0] if weights else Wi).T + h0 @ (weights[1] if weights else Wh).T + b
    E = tau * (feat.abs() @ Wi.abs().T + h0.abs() @ Wh.abs().T + lstm.bias_ih_l0.abs() + lstm.bias_hh_l0.abs()) + ALPHA
    zi, zf, zg, zo = z.chunk(4, 1)
    Ei, Ef, Eg, Eo = E.chunk(4, 1)
    i, f, g, o = torch.sigmoid(zi), torch.sigmoid(zf), torch.tanh(zg), torch.sigmoid(zo)
    c1 = f * c0 + i * g
    h1 = o * torch.tanh(c1)
    ec = (Ef / 4 + EXPF_ERR) * c0.abs() + (Ei / 4 + EXPF_ERR) * g.abs() + i * (Eg + EXPF_ERR) + ALPHA
    eh = (Eo / 4 + EXPF_ERR) * torch.tanh(c1).abs() + o * (ec + EXPF_ERR) + ALPHA
    return h1, c1, eh, ec


@pytest.mark.parametrize("hc", [16, 8])
def test_efficientzero_trunk_features_and_lstm(hc):
    """EfficientZero: the trunk layers and the reward features through the hook; the LSTM h / c of
    recurrent_inference against a float64 nn.LSTM step on those features.  hc = 16: nin = 576 (k_ez_lstm_tc),
    hc = 8: nin = 288 (the fp32 k_ez_lstm)."""
    A, B = 6, 397
    ref64, cu = make_models(A=A, hc=(hc, 16, 16), seed=40 + hc, ez=True)
    # latents of at most 3: the LSTM gates then span the sigmoid / tanh instead of saturating
    latent, action = make_latents(B, seed=hc, peak=3.0), (torch.arange(B) % A).cuda()
    for which in (0, 1):
        ratios, _, out, _ = run_program(cu, ref64, which, latent, action)
        assert max(ratios.values()) <= 1.0, ratios
        if which == 0:
            assert "ez_feat" in ratios
            feat = out["feat"].double()
        check_scalars(out, which, True)
    H = cu.lstm_hidden_size
    g = torch.Generator().manual_seed(hc)
    h0 = (0.5 * torch.randn(B, H, generator=g)).cuda()
    c0 = (2.0 * torch.randn(B, H, generator=g)).cuda()
    o = cu.recurrent_inference(latent, (h0[None], c0[None]), action)
    with torch.no_grad():
        h1, c1, eh, ec = lstm_bound(ref64.dynamics_network.lstm, feat, h0.double(), c0.double())
    nh, nc = o.reward_hidden_state
    rh, rc = worst(nh[0].double() - h1, eh), worst(nc[0].double() - c1, ec)
    assert rh <= 1.0 and rc <= 1.0, (rh, rc)
