"""The tensor-core DownSample tower launch by launch against float64 (lz_model_debug_tower_stage).

Each stage's reference runs on exactly the operands that launch consumed: the hi + lo sum of the previous stage's dump,
summed in float64.  A stage's error is then that launch's alone, and it is compared element by element with

    |y_cuda - y_f64| <= TAU[stage] * M + ALPHA * S

M is the same stage evaluated in float64 on |W|, |x|, the BatchNorm terms |scale| (|conv| + |mean|) + |beta| and |residual|,
so the bound does not depend on cancellation or on the scale of a layer.  S = |scale| (|W| (*) S_in) + 1 counts the
operands whose fp16 lo part can be subnormal (absolute error 2^-25 each): the conv1 output a fused ResBlock keeps in shared
memory, and the stored output itself.

Error analysis of one 3xFP16 stage (u = 2^-24): the input x = x_hi + x_lo is exact; the weights carry the 2^-22 relative
residual of their hi/lo split; the dropped x_lo * w_lo product is <= 2^-22 |x| |w|; the tensor cores accumulate in fp32;
the folded BatchNorm carries a few fp32 roundings; the hi/lo split of the output keeps 22 bits (2^-22 relative).  That puts
a few 2^-22 of M on every wgmma stage, twice for a fused ResBlock, and TAU is that figure calibrated on an H100 so that the
3xFP16 build stays under a quarter of the bound.  A single fp16 pass (tc1) drops x_lo * w_hi and x_hi * w_lo, 2^-11
relative per product: test_stage_bound_detects_single_pass proves that the bound sees that.
"""
import copy

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

WGMMA_STAGES = (1, 2, 3, 4, 5, 7)
STAGE_NAMES = ("stem", "resblocks1", "ds.conv1", "ds.conv3", "ds.conv2+id", "resblocks2", "pool1", "resblocks3", "pool2")
# calibrated per stage (DESIGN.md 4.3): the worst tc3 element stays <= 1/4 of the bound, the worst tc1 element of every
# wgmma stage exceeds it by >= 8x
TAU = (2.0 ** -19, 2.0 ** -21, 2.0 ** -17, 2.0 ** -17, 2.0 ** -18, 2.0 ** -21, 2.0 ** -19, 2.0 ** -22, 2.0 ** -19)
ALPHA = 2.0 ** -23
MAX_IMG_BYTES = 512 * 1024          # >= the largest tower tensor of one 96-px image
N_SMS = 132


# ------------------------------------------------------------------------------------------------ models and inputs
def _models(obs=(4, 84, 84), A=18, seed=21, math="tc3", mutate=None):
    import lightzero_b200 as lzb
    from oracle.model_ref import MuZeroModelRef, emulate_trained_
    torch.manual_seed(seed)
    ref = emulate_trained_(MuZeroModelRef(obs, A), seed)
    if mutate is not None:
        mutate(ref)
    cu = lzb.MuZeroModel(observation_shape=obs, action_space_size=A).load_state_dict(ref.state_dict())
    cu.set_math(math)
    ref64 = copy.deepcopy(ref).double().cuda().eval()
    return ref, ref64, cu


def _atari_frames(B, C, px, seed):
    """uint8 frames like an Atari screen: a constant background per frame with a few sparse bright objects; the batch
    also holds an all-0 and an all-255 frame (dead-ReLU regions and the largest scaled input)."""
    g = np.random.default_rng(seed)
    x = np.empty((B, C, px, px), np.uint8)
    for b in range(B):
        x[b] = g.choice([0, 17, 74, 142])
        for _ in range(g.integers(2, 9)):
            h, w = g.integers(2, 10, size=2)
            y0, x0 = g.integers(0, px - h), g.integers(0, px - w)
            x[b, :, y0:y0 + h, x0:x0 + w] = g.integers(160, 256, size=(C, 1, 1))
    if B >= 3:
        x[0] = 0
        x[1] = 255
    return torch.from_numpy(x)


def _inputs(kind, B, C, px, seed):
    """(device tensor handed to the CUDA tower, the float64 values its stem reads)"""
    if kind == "float":
        x = torch.rand(B, C, px, px, generator=torch.Generator().manual_seed(seed)).cuda()
        return x, x.double()
    u8 = _atari_frames(B, C, px, seed).cuda()
    return u8, (u8.double() / 255.0).float().double()      # the stem divides in fp32, correctly rounded


# ------------------------------------------------------------------------------------------------ the hook and TCL decoding
def dump_stage(cu, obs, stage):
    """(raw bytes of the stage's output tensor, h_info)"""
    from lightzero_b200 import cabi
    B = obs.shape[0]
    buf = torch.empty(B * MAX_IMG_BYTES, dtype=torch.uint8, device="cuda")
    info = np.zeros(10, np.int32)
    f32 = obs if obs.dtype == torch.float32 else None
    u8 = obs if obs.dtype == torch.uint8 else None
    cabi.check(cu._lib.lz_model_debug_tower_stage(cu._h, B, cabi.ptr(f32), cabi.ptr(u8), stage, buf.data_ptr(), buf.numel(),
                                                  info.ctypes.data, cabi.stream_ptr()), "lz_model_debug_tower_stage")
    torch.cuda.synchronize()
    info = [int(v) for v in info]
    return buf[:B * image_bytes(info)], info


def image_bytes(info):
    C, H, W, nph, R = info[:5]
    return C * H * W * 4 if nph == 0 else nph * 2 * (C // 8) * R * 16


def tcl_halves(raw, info, B):
    """raw TCL bytes -> fp16 [B][nphase][hi|lo][C][plane_rows]"""
    C, _, _, nph, R = info[:5]
    h = raw.view(torch.float16).reshape(B, nph, 2, C // 8, R, 8)
    return h.permute(0, 1, 2, 3, 5, 4).reshape(B, nph, 2, C, R)


def tcl_grid(raw, info, B):
    """fp16 [B][nphase][hi|lo][C][H + 2][pitch]: the padded grid (rows 1 .. R - 2 of every plane)"""
    _, H, _, _, R = info[:5]
    pitch = (R - 2) // (H + 2)
    assert (H + 2) * pitch + 2 == R and pitch > info[2], info
    return tcl_halves(raw, info, B)[..., 1:R - 1].reshape(*tcl_halves(raw, info, B).shape[:4], H + 2, pitch)


def stage_value(raw, info, B):
    """float64 NCHW image of a stage's output (hi + lo; phase-split tensors re-interleaved)"""
    C, H, W, nph, _ = info[:5]
    if nph == 0:
        return raw.view(torch.float32).reshape(B, C, H, W).double()
    g = tcl_grid(raw, info, B)
    v = g[:, :, 0, :, 1:H + 1, :W].double() + g[:, :, 1, :, 1:H + 1, :W].double()
    if nph == 1:
        return v[:, 0]
    out = torch.empty(B, C, 2 * H, 2 * W, dtype=torch.float64, device=v.device)
    for f in range(4):
        out[:, :, f >> 1::2, f & 1::2] = v[:, f]
    return out


# ------------------------------------------------------------------------------------------------ float64 references
def _conv(conv, bn, x, M, S, relu):
    """conv (+ BatchNorm) (+ ReLU) on (value, magnitude, subnormal count); BN in its eval form s (z - mean) + beta"""
    kw = dict(stride=conv.stride, padding=conv.padding)
    y = F.conv2d(x, conv.weight, **kw)
    Wa = conv.weight.abs()
    M, S = F.conv2d(M, Wa, **kw), F.conv2d(S, Wa, **kw)
    if bn is not None:
        s = (bn.weight / torch.sqrt(bn.running_var + bn.eps)).view(1, -1, 1, 1)
        mean, beta = bn.running_mean.view(1, -1, 1, 1), bn.bias.view(1, -1, 1, 1)
        y = s * (y - mean) + beta
        M = s.abs() * (M + mean.abs()) + beta.abs()
        S = s.abs() * S
    return (torch.relu(y) if relu else y), M, S + 1.0


def _resblock(blk, x):
    t, Mt, St = _conv(blk.conv1[0], blk.conv1[1], x, x.abs(), torch.zeros_like(x), True)
    y, M, S = _conv(blk.conv2[0], blk.conv2[1], t, Mt, St, False)
    return torch.relu(y + x), M + x.abs(), S


def _pool(x):
    p = lambda v: F.avg_pool2d(v, 3, 2, 1, count_include_pad=True)
    return p(x), p(x.abs()), torch.ones_like(p(x))


def stage_reference(ds, stage, x, x2=None):
    """(y, M, S) of one tower stage in float64 on the stage's own inputs x (and x2 = U1 for stage 4)"""
    z = torch.zeros_like(x)
    if stage == 0:
        return _conv(ds.conv1, ds.norm1, x, x.abs(), z, True)
    if stage == 1:
        return _resblock(ds.resblocks1[0], x)
    db = ds.downsample_block
    if stage == 2:
        return _conv(db.conv1[0], db.conv1[1], x, x.abs(), z, True)
    if stage == 3:
        return _conv(db.conv3[0], None, x, x.abs(), z, False)
    if stage == 4:
        y, M, S = _conv(db.conv2[0], db.conv2[1], x, x.abs(), z, False)
        return torch.relu(y + x2), M + x2.abs(), S
    if stage == 5:
        return _resblock(ds.resblocks2[0], x)
    if stage == 7:
        return _resblock(ds.resblocks3[0], x)
    return _pool(x)


def stage_ratios(cu, ref64, obs, x64):
    """per stage: worst |err| / (TAU M + ALPHA S), raw dump, info, largest |float64 reference|; each stage is checked on
    the CUDA's own input"""
    ds = ref64.representation_network.downsample_net
    B = obs.shape[0]
    raws, infos, vals, out, peaks = [], [], [], [], []
    for st in range(9):
        raw, info = dump_stage(cu, obs, st)
        raws.append(raw)
        infos.append(info)
        vals.append(stage_value(raw, info, B))
    inputs = {0: (x64,), 1: (vals[0],), 2: (vals[1],), 3: (vals[1],), 4: (vals[2], vals[3]), 5: (vals[4],), 6: (vals[5],),
              7: (vals[6],), 8: (vals[7],)}
    with torch.no_grad():
        for st in range(9):
            y, M, S = stage_reference(ds, st, *inputs[st])
            assert y.shape == vals[st].shape, (st, y.shape, vals[st].shape)
            out.append(((vals[st] - y).abs() / (TAU[st] * M + ALPHA * S)).max().item())
            peaks.append(y.abs().max().item())
    return out, raws, infos, peaks


# ------------------------------------------------------------------------------------------------ TCL invariants
def tcl_violations(raw, info, B):
    """counts of: non-zero pad / spare entries, invalid (hi, lo) splits, non-finite halves"""
    C, H, W, nph, R = info[:5]
    halves = tcl_halves(raw, info, B)
    grid = tcl_grid(raw, info, B)
    pad = (halves[..., 0] != 0).sum() + (halves[..., R - 1] != 0).sum()           # the spare rows
    pad += (grid[..., 0, :] != 0).sum() + (grid[..., H + 1, :] != 0).sum()         # the pad rows above / below
    pad += (grid[..., 1:H + 1, W:] != 0).sum()                                     # the pad column
    hi = halves[:, :, 0].cpu().numpy().ravel()
    lo = halves[:, :, 1].cpu().numpy().ravel()
    finite = np.isfinite(hi) & np.isfinite(lo)
    # gap: the distance from hi to its fp16 neighbour on lo's side.  hi = rn(v) and lo = rn(v - hi) can round lo onto
    # exactly gap / 2 with an odd hi (v - hi was just under the half gap), so hi == rn(hi + lo) holds except at such ties
    lo64 = lo.astype(np.float64)
    gap = np.abs(np.nextafter(hi, np.where(lo < 0, np.float16(-np.inf), np.float16(np.inf))).astype(np.float64) - hi)
    split_ok = (np.abs(lo64) <= gap / 2) & (((hi.astype(np.float64) + lo64).astype(np.float16) == hi) | (np.abs(lo64) == gap / 2))
    return int(pad.item()), int((~split_ok & finite).sum()), int((~finite).sum())


# ------------------------------------------------------------------------------------------------ tests
_CASES = {}


def _case(px, kind, B):
    """one model per (px, input, B): every stage's worst ratio, TCL invariant counts and plan"""
    key = (px, kind, B)
    if key not in _CASES:
        _, ref64, cu = _models((4, px, px))
        obs, x64 = _inputs(kind, B, 4, px, seed=px + B)
        ratios, raws, infos, _ = stage_ratios(cu, ref64, obs, x64)
        inv = [tcl_violations(raws[st], infos[st], B) if infos[st][3] else (0, 0, 0) for st in range(9)]
        _CASES[key] = (ratios, inv, infos)
        del raws
        torch.cuda.empty_cache()
    return _CASES[key]


PX, KINDS, BATCHES = (84, 96), ("float", "uint8"), (1, 3, 131, 1024)


@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("px", PX)
def test_stage_matches_float64(px, kind, B):
    ratios, _, _ = _case(px, kind, B)
    bad = {STAGE_NAMES[st]: r for st, r in enumerate(ratios) if not r <= 1.0}
    assert not bad, f"stages over the float64 bound (worst |err| / bound): {bad}"


@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("px", PX)
def test_tcl_invariants(px, kind, B):
    _, inv, infos = _case(px, kind, B)
    for st in range(8):
        assert infos[st][3] in (1, 4) and (st == 1) == (infos[st][3] == 4), infos[st]
        pad, split, nonfinite = inv[st]
        assert (pad, split, nonfinite) == (0, 0, 0), \
            f"{STAGE_NAMES[st]}: {pad} non-zero pad entries, {split} invalid hi/lo splits, {nonfinite} NaN/Inf"


@pytest.mark.parametrize("px", PX)
def test_stage_bound_detects_single_pass(px):
    """The same bound must fail a single fp16 pass by >= 8x on every wgmma stage: it can see a dropped hi/lo pass."""
    _, ref64, cu = _models((4, px, px), math="tc1")
    obs, x64 = _inputs("float", 131, 4, px, seed=3)
    ratios, _, infos, _ = stage_ratios(cu, ref64, obs, x64)
    assert all(infos[st][9] == 1 for st in range(9))
    weak = {STAGE_NAMES[st]: ratios[st] for st in WGMMA_STAGES if not ratios[st] >= 8.0}
    assert not weak, f"tc1 within 8x of the bound (worst |err| / bound): {weak}"


def test_plan_edges_are_covered():
    """The sizes above must include a launch with a short last band, one with a partial image group and a grid of more
    than one wave: if a plan change loses one, pick another px or B rather than lose the coverage."""
    short_band = partial_group = multi_wave = None
    for px in PX:
        _, _, cu = _models((4, px, px))
        for B in BATCHES:
            obs = torch.zeros(B, 4, px, px, device="cuda")
            for st in WGMMA_STAGES:
                C, H, W, nph, R, G, bh, stages, ctas, npass = dump_stage(cu, obs, st)[1]
                assert npass == 3 and 2 <= stages <= 4 and G >= 1 and bh >= 1
                Hrows = 2 * H if st == 1 else H                      # resblocks1 writes the phase split of a 2H image
                if G == 1 and Hrows % bh != 0:
                    short_band = short_band or (px, B, STAGE_NAMES[st], Hrows, bh)
                if G > 1 and B % G != 0:
                    partial_group = partial_group or (px, B, STAGE_NAMES[st], G)
                if st in (1, 5, 7) and ctas > N_SMS:                # the fused ResBlock runs one CTA per SM
                    multi_wave = multi_wave or (px, B, STAGE_NAMES[st], ctas)
    assert short_band and partial_group and multi_wave, (short_band, partial_group, multi_wave)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("C", [3, 9])
def test_other_observation_channels(C, kind):
    """Observations with != 4 channels take the k_conv3x3_generic stem (9 channels: a chunk of 8 and a remainder of 1)."""
    B, px = 131, 84
    _, ref64, cu = _models((C, px, px), A=6, seed=C)
    obs, x64 = _inputs(kind, B, C, px, seed=C)
    ds = ref64.representation_network.downsample_net
    raw, info = dump_stage(cu, obs, 0)
    with torch.no_grad():
        y, M, S = stage_reference(ds, 0, x64)
    r = ((stage_value(raw, info, B) - y).abs() / (TAU[0] * M + ALPHA * S)).max().item()
    assert r <= 1.0, r
    assert tcl_violations(raw, info, B) == (0, 0, 0)
    if kind == "float":
        out = cu.initial_inference(obs)
        with torch.no_grad():
            exp = ref64.initial_inference(x64)
        for a, e in ((out.latent_state, exp.latent_state), (out.policy_logits, exp.policy_logits), (out.value, exp.value)):
            assert torch.allclose(a.double(), e, rtol=1e-5, atol=1e-5), (a.double() - e).abs().max().item()
    else:
        # uint8 frames reach initial_inference through the tower only (the search collectors); the whole tower suffices
        raw8, info8 = dump_stage(cu, obs, 8)
        ratios, _, _, _ = stage_ratios(cu, ref64, obs, x64)
        assert max(ratios) <= 1.0, ratios
        with torch.no_grad():
            pre = ds(x64)
        assert torch.allclose(stage_value(raw8, info8, B), pre, rtol=1e-5, atol=1e-5)


def _dynamic_range(ref):
    """per-output-channel conv weight multipliers 2^-10 .. 2^3, BatchNorm running_var down to 1e-4 (on the channels whose
    weights are small, so that activations stay inside the fp16 range)"""
    g = torch.Generator().manual_seed(7)
    ds = ref.representation_network.downsample_net
    with torch.no_grad():
        for mod in ds.modules():
            if not isinstance(mod, torch.nn.Conv2d):
                continue
            co = mod.weight.shape[0]
            e = torch.linspace(-10.0, 3.0, co)[torch.randperm(co, generator=g)]
            mod.weight.mul_((2.0 ** e).view(-1, 1, 1, 1))
            mod._lz_exp = e
        for blk in list(ds.resblocks1) + [ds.downsample_block] + list(ds.resblocks2) + list(ds.resblocks3):
            for seq in (blk.conv1, blk.conv2):
                conv, bn = seq[0], seq[1]
                small = conv._lz_exp <= -2
                bn.running_var[small] = 1e-4 * (1.0 + torch.rand(int(small.sum()), generator=g))
        ds.norm1.running_var[ds.conv1._lz_exp <= -2] = 1e-4
    for mod in ds.modules():
        if hasattr(mod, "_lz_exp"):
            del mod._lz_exp


def test_dynamic_range():
    """A layer's one power-of-two weight scale leaves small channels with fp16-subnormal lo parts; small BatchNorm variances
    push activations towards the fp16 maximum (65504, where the hi/lo split clamps)."""
    px, B = 84, 131
    _, ref64, cu = _models((4, px, px), mutate=_dynamic_range)
    obs, x64 = _inputs("float", B, 4, px, seed=9)
    ratios, raws, infos, vmax = stage_ratios(cu, ref64, obs, x64)
    assert 1e3 < max(vmax) < 6e4, dict(zip(STAGE_NAMES, vmax))      # near the fp16 maximum, inside it
    assert max(ratios) <= 1.0, dict(zip(STAGE_NAMES, ratios))
    for st in range(8):
        assert tcl_violations(raws[st], infos[st], B) == (0, 0, 0), STAGE_NAMES[st]


def _all_stages(cu, obs):
    return [dump_stage(cu, obs, st)[0].clone() for st in range(9)]


def test_workspace_reuse_and_batch_position():
    """Per-row sums keep one tap -> k-step -> pass order whatever the band or group an image lands in (DESIGN.md 4.3), so
    the stage outputs of an image are bit-identical across batch sizes, workspace histories and batch positions."""
    px = 84
    X = torch.rand(1024, 4, px, px, generator=torch.Generator().manual_seed(1)).cuda()
    Y = torch.rand(131, 4, px, px, generator=torch.Generator().manual_seed(2)).cuda()
    Yu8 = _atari_frames(131, 4, px, 3).cuda()
    fresh_Y = _all_stages(_models((4, px, px))[2], Y)
    fresh_X = _all_stages(_models((4, px, px))[2], X)
    fresh_Yu8 = _all_stages(_models((4, px, px))[2], Yu8)
    # a large batch, then a small one in the same workspace
    _, _, cu = _models((4, px, px))
    _all_stages(cu, X)
    assert all(torch.equal(a, b) for a, b in zip(_all_stages(cu, Y), fresh_Y))
    # the reverse order grows the workspace
    _, _, cu = _models((4, px, px))
    _all_stages(cu, Y)
    assert all(torch.equal(a, b) for a, b in zip(_all_stages(cu, X), fresh_X))
    # float and uint8 calls interleaved
    _, _, cu = _models((4, px, px))
    for obs, exp in ((Yu8, fresh_Yu8), (Y, fresh_Y), (Yu8, fresh_Yu8), (Y, fresh_Y)):
        assert all(torch.equal(a, b) for a, b in zip(_all_stages(cu, obs), exp))
    # batch position: a permuted batch, and one image alone
    perm = torch.randperm(131, generator=torch.Generator().manual_seed(4)).cuda()
    permuted = _all_stages(cu, Y[perm].contiguous())
    for st in range(9):
        n = fresh_Y[st].numel() // 131
        a, b = permuted[st].view(131, n), fresh_Y[st].view(131, n)[perm]
        assert torch.equal(a, b), STAGE_NAMES[st]
    for j in (0, 77, 130):
        single = _all_stages(cu, Y[j:j + 1].contiguous())
        for st in range(9):
            n = single[st].numel()
            assert torch.equal(single[st], fresh_Y[st].view(131, n)[j]), (j, STAGE_NAMES[st])


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


@pytest.mark.parametrize("math,px", [pytest.param("tc3", 84, id="tc3"), pytest.param("tc3", 96, id="tc3_96px")])
def test_recurrent_on_search_latents(math, px):
    """recurrent_inference on what a search feeds it: sparse post-ReLU latents, chained up to S steps deep, against float64.
    Latents and logits at 1e-5, scalars at 2e-4 (DESIGN.md 4.4)."""
    import lightzero_b200 as lzb
    from oracle.model_ref import DiscreteSupport, InverseScalarTransform
    B, A, S = 300, 18, 50
    _, ref64, cu = _models((4, px, px), A=A, seed=31, math=math)
    rng = np.random.default_rng(0)
    obs = torch.rand(B, 4, px, px, generator=torch.Generator().manual_seed(5)).cuda()
    out = cu.initial_inference(obs)
    legal = [list(range(A))] * B
    noises = [rng.dirichlet([0.3] * A).astype(np.float32).tolist() for _ in range(B)]
    mcts = lzb.MuZeroMCTSCtree(dict(num_simulations=S, deterministic=True, discount_factor=0.997))
    roots = mcts.roots(B, legal)
    roots.prepare(0.25, noises, [0.] * B, out.policy_logits, [-1] * B)
    rec = _Recorder(cu)
    mcts.search(roots, rec, out.latent_state, [-1] * B)
    assert len(rec.calls) == S
    inv = InverseScalarTransform(DiscreteSupport(-300., 301., 1.))
    zero_frac = []
    for latent, action, o in rec.calls:
        with torch.no_grad():
            exp = ref64.recurrent_inference(latent.double(), action.reshape(-1).long())
        zero_frac.append((latent == 0).double().mean().item())
        for a, e in ((o.latent_state, exp.latent_state), (o.reward, exp.reward), (o.value, exp.value),
                     (o.policy_logits, exp.policy_logits)):
            assert torch.allclose(a.double(), e, rtol=1e-5, atol=1e-5), (a.double() - e).abs().max().item()
        with torch.no_grad():
            ev, er = inv(exp.value.float().cpu()).reshape(-1), inv(exp.reward.float().cpu()).reshape(-1)
        assert torch.allclose(o.value_scalar.cpu(), ev, rtol=2e-4, atol=2e-4)
        assert torch.allclose(o.reward_scalar.cpu(), er, rtol=2e-4, atol=2e-4)
    assert min(zero_frac) > 0.05, zero_frac       # the latents are post-ReLU and sparse
    roots.clear()
