"""64x64 observations (the shipped Atari configs of MuZero and EfficientZero: DownSample to an 8x8 latent, no pooling2).

The latent-grid kernel runs its 8x8 instantiation (4 roots per CTA, FC1 over 1,024 inputs as m64n32); the DownSample tower
ends in a TCL -> NCHW conversion instead of pooling2.  Checked here:
- initial / recurrent inference against the PyTorch restatement at 1e-5 (scalars at 2e-4) over every CTA packing;
- every layer and head of both programs against float64 under the |y - y64| <= TAU M + ALPHA S bound of
  test_gpu_net_layers.py, which a single fp16 pass (tc1) must exceed;
- every tower stage against float64 (stage 8, the conversion, bit for bit against hi + lo of stage 7);
- root outputs independent of the root's slot and packing;
- the CUDA models against the reference-class fixtures tests/golden/obs64_*.npz at 1e-5;
- the fused searches against the oracle driving the same network, the step-wise drives, uint8 frames, and refusals.
"""
import copy
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_gpu_net_layers import ALPHA, SUPPORT, TAU, check_scalars, head_features, head_reference, inverse_h, layer_reference, \
    lstm_bound, program, split_full, split_hi_lo, worst
from oracle.tree_drive import assert_same
from test_gpu_search_oracle import _inputs as search_inputs, fused_search, oracle_search
from test_gpu_tower_layers import ALPHA as T_ALPHA, TAU as T_TAU, WGMMA_STAGES, _atari_frames, dump_stage, stage_reference, \
    stage_value, tcl_grid

from conftest import GOLDEN_DIR, ROOT

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

OBS = (4, 64, 64)
HW, P = 8, 64
N_SMS = 132


def make_models(A=6, nres=1, hc=(16, 16, 16), seed=0, math="tc3", ez=False):
    """(fp32 restatement on the CPU, float64 copy on the GPU, CUDA model) at 64x64"""
    import lightzero_b200 as lzb
    from oracle.model_ref import EfficientZeroModelRef, MuZeroModelRef, emulate_trained_
    torch.manual_seed(seed)
    kw = dict(num_res_blocks=nres, reward_head_channels=hc[0], value_head_channels=hc[1], policy_head_channels=hc[2])
    ref = emulate_trained_((EfficientZeroModelRef if ez else MuZeroModelRef)(OBS, A, **kw), seed)
    cu = (lzb.EfficientZeroModel if ez else lzb.MuZeroModel)(observation_shape=OBS, action_space_size=A, downsample=True, **kw)
    cu.load_state_dict(ref.state_dict())
    cu.set_math(math)
    return ref, copy.deepcopy(ref).double().cuda().eval(), cu


def make_latents(B, seed, peak=None):
    g = torch.Generator().manual_seed(seed)
    x = torch.relu(torch.randn(B, 64, HW, HW, generator=g))
    s = torch.tensor((0.0, 1e-3, 0.05, 1.0, 1.0, 4.0, 30.0, 2e3))[torch.randint(0, 8, (B,), generator=g)]
    x = x * s.view(-1, 1, 1, 1)
    if peak is not None and x.max() > 0:
        x = x * (peak / x.max())
    return x.cuda()


def pick_roots(B):
    """tc_pick_roots on the 8x8 grid: one wave of one CTA per SM, at most 4 roots (3 row tiles)"""
    return min(max(-(-B // N_SMS), 1), 4)


# ------------------------------------------------------------------------------------------------ restatement parity
PARITY = [(B, A, nres) for B, A, nres in ((1, 6, 1), (3, 18, 2), (4, 6, 1), (5, 18, 1), (131, 6, 2), (1024, 18, 1), (1201, 6, 1))]


@pytest.mark.parametrize("B,A,nres", PARITY)
def test_inference_matches_restatement(B, A, nres):
    ref, _, cu = make_models(A=A, nres=nres, seed=B + A)
    obs = torch.rand((B,) + OBS, generator=torch.Generator().manual_seed(B))
    action = torch.randint(0, A, (B,), generator=torch.Generator().manual_seed(B + 1))
    assert cu.latent_hw == HW
    with torch.no_grad():
        e0 = ref.initial_inference(obs)
        o0 = cu.initial_inference(obs.cuda())
        for f in ("policy_logits", "latent_state", "value"):
            assert torch.allclose(getattr(o0, f).cpu(), getattr(e0, f), rtol=1e-5, atol=1e-5), f
        assert o0.latent_state.shape == (B, 64, HW, HW)
        e1 = ref.recurrent_inference(e0.latent_state, action)
        o1 = cu.recurrent_inference(e0.latent_state.cuda(), action.cuda(), return_scalars=True)
        for f in ("policy_logits", "latent_state", "value", "reward"):
            assert torch.allclose(getattr(o1, f).cpu(), getattr(e1, f), rtol=1e-5, atol=1e-5), f
        for f, logits in (("value_scalar", e1.value), ("reward_scalar", e1.reward)):
            exp = inverse_h(logits.double(), SUPPORT).float()
            assert torch.allclose(getattr(o1, f).cpu().reshape(-1), exp, rtol=0, atol=2e-4 * max(1.0, exp.abs().max().item())), f
    cu.set_math("tc1")          # the fast single-pass mode runs at every size too
    o = cu.recurrent_inference(e0.latent_state.cuda(), action.cuda())
    assert torch.isfinite(o.policy_logits).all() and torch.isfinite(o.latent_state).all()
    assert torch.isfinite(cu.initial_inference(obs.cuda()).value).all()


FIXTURES = ("obs64_muzero_a6", "obs64_ez_a6", "obs64_muzero_a18_r2")


@pytest.mark.parametrize("name", FIXTURES)
def test_cuda_model_matches_reference_class_vectors(name):
    """tests/golden/obs64_*.npz, written by make_obs64_golden.py from the REFERENCE'S OWN model classes at 64x64; the
    weights are regenerated from the fixture's seed through the restatement (checked by SHA-256)"""
    import lightzero_b200 as lzb
    from make_model_golden import build_restated, weights_digest
    d = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    kind, A, nres = str(d["kind"]), int(d["A"]), int(d["nres"])
    ref = build_restated(kind, OBS, A, nres, int(d["seed"]))
    if weights_digest(ref) != str(d["weights_sha256"]):
        pytest.skip("this torch build initialises parameters differently from the one that wrote the fixture")
    cls = lzb.EfficientZeroModel if kind == "efficientzero" else lzb.MuZeroModel
    cu = cls(observation_shape=OBS, action_space_size=A, num_res_blocks=nres, downsample=True).load_state_dict(ref.state_dict())
    tol = dict(rtol=1e-5, atol=1e-5)
    obs, action = torch.from_numpy(d["obs"]).cuda(), torch.from_numpy(d["action"]).cuda()
    o0 = cu.initial_inference(obs)
    for f in ("value", "policy_logits", "latent_state"):
        assert torch.allclose(getattr(o0, f).cpu(), torch.from_numpy(d["init_" + f]), **tol), (name, "initial", f)
    latent = torch.from_numpy(d["init_latent_state"]).cuda()
    if kind == "efficientzero":
        hc = (torch.from_numpy(d["in_hidden0"]).cuda(), torch.from_numpy(d["in_hidden1"]).cuda())
        o1 = cu.recurrent_inference(latent, hc, action)
        for f in ("value", "value_prefix", "policy_logits", "latent_state"):
            assert torch.allclose(getattr(o1, f).cpu(), torch.from_numpy(d["rec_" + f]), **tol), (name, "recurrent", f)
        for i in range(2):
            assert torch.allclose(o1.reward_hidden_state[i].cpu(), torch.from_numpy(d[f"rec_hidden{i}"]), **tol), (name, "hidden", i)
    else:
        o1 = cu.recurrent_inference(latent, action)
        for f in ("value", "reward", "policy_logits", "latent_state"):
            assert torch.allclose(getattr(o1, f).cpu(), torch.from_numpy(d["rec_" + f]), **tol), (name, "recurrent", f)


# ------------------------------------------------------------------------------------------------ layer by layer
def net_stage(cu, which, latent, action, stage, nlayers):
    from lightzero_b200 import cabi
    B, K, A = latent.shape[0], cu.value_support_size, cu.action_space_size
    nfeat = cu._cfg.reward_head_channels * P if cu._cfg.efficientzero else 0
    n = B * 64 * P if stage < nlayers else B * (2 * K + 2 * A + 4 + nfeat)
    buf = torch.full((n,), float("nan"), dtype=torch.float32, device="cuda")
    info = np.zeros(8, np.int32)
    act = action.to(torch.int32).contiguous() if action is not None else None
    cabi.check(cu._lib.lz_model_debug_net_stage(cu._h, which, B, latent.contiguous().data_ptr(), cabi.ptr(act), stage,
                                                buf.data_ptr(), buf.numel() * 4, info.ctypes.data, cabi.stream_ptr()),
               "lz_model_debug_net_stage")
    torch.cuda.synchronize()
    return buf, [int(v) for v in info]


def run_program(cu, ref64, which, latent, action):
    """{stage: worst |err| / bound} of every layer and head of one program, the full outputs and the plans"""
    layers, rew_hook = program(ref64, which)
    nl, B, A = len(layers), latent.shape[0], cu.action_space_size
    ez = bool(cu._cfg.efficientzero)
    dumps, infos = [], []
    for L in range(nl):
        buf, info = net_stage(cu, which, latent, action, L, nl)
        dumps.append(buf.view(B, 64, HW, HW).double())
        infos.append(info)
    buf, info = net_stage(cu, which, latent, action, nl, nl)
    infos.append(info)
    out = split_full(buf, B, cu.value_support_size, A, cu._cfg.reward_head_channels * P if ez else 0)
    x0 = latent.double()
    onehot = F.one_hot(action.long(), A).double().view(B, A, 1, 1).expand(B, A, HW, HW) if which == 0 else None
    ratios = {}
    with torch.no_grad():
        for L, (conv, bn, kind) in enumerate(layers):
            res = x0 if kind == "dyn" else ((dumps[L - 2] if L >= 2 else x0) if kind == "conv2" else None)
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
            ratios[f"{name} head"] = worst(got.double() - y, TAU[name] * M + ALPHA * S)
        if which == 0 and ez:
            f, Mf = head_features(dyn.conv1x1_reward, dyn.norm_reward, split_hi_lo(dumps[rew_hook]))
            ratios["ez_feat"] = worst(out["feat"].double() - f, TAU["feat"] * Mf + ALPHA)
    return ratios, out, infos


def check_plan(info, B, nlayers):
    R = pick_roots(B)
    ctas = -(-B // R)
    assert info[:6] == [R, (81 * R - 10 + 127) >> 7, ctas, B - (ctas - 1) * R, nlayers, 3], (B, info)
    assert info[0] <= 4 and info[1] <= 3


# (A, num_res_blocks, head channels): FC1 over 1024 / 512 / 64 inputs
NET_CONFIGS = [(18, 1, (16, 16, 16)), (6, 2, (8, 1, 16)), (33, 1, (1, 16, 8))]
NET_B = (1, 3, 4, 5, 131, 133, 266, 397, 1024, 1201)


@pytest.mark.parametrize("cfg", NET_CONFIGS, ids=lambda c: f"A{c[0]}-nres{c[1]}-hc{'.'.join(map(str, c[2]))}")
def test_layers_match_float64(cfg):
    A, nres, hc = cfg
    _, ref64, cu = make_models(A=A, nres=nres, hc=hc, seed=A + nres)
    for which in (0, 1):
        for B in NET_B:
            latent = make_latents(B, seed=B + which)
            action = (torch.arange(B) % A).cuda()
            ratios, out, infos = run_program(cu, ref64, which, latent, action)
            bad = {k: r for k, r in ratios.items() if not r <= 1.0}
            assert not bad, f"which={which} B={B}: over the float64 bound: {bad}"
            check_scalars(out, which, False)
            nl = len(infos) - 1
            for L, info in enumerate(infos):
                check_plan(info, B, min(L + 1, nl))
    packings = {(pick_roots(B), B - (-(-B // pick_roots(B)) - 1) * pick_roots(B)) for B in NET_B}
    assert {R for R, _ in packings} == {1, 2, 3, 4} and any(1 < last < R for R, last in packings)


def test_bound_detects_single_pass():
    _, ref64, cu = make_models(A=18, seed=5, math="tc1")
    B = 131
    latent, action = make_latents(B, seed=7), (torch.arange(B) % 18).cuda()
    for which in (0, 1):
        ratios, _, _ = run_program(cu, ref64, which, latent, action)
        assert min(ratios.values()) > 1.0, ratios


def test_root_outputs_identical_at_every_slot_and_packing():
    """a root's outputs do not depend on the batch it runs in (R = 1 ... 4, its slot in the CTA, a second wave)"""
    _, _, cu = make_models(A=18, seed=9)
    base = make_latents(8, seed=3)
    act = (torch.arange(8) % 18).cuda()
    ref = cu.recurrent_inference(base, act, return_scalars=True)
    for B in (8, 131, 263, 397, 530, 1201):
        for off in (0, 1, 2, 3):
            if off + 8 > B:
                continue
            lat = make_latents(B, seed=B + off)
            a = (torch.arange(B) % 18).cuda()
            lat[off:off + 8], a[off:off + 8] = base, act
            o = cu.recurrent_inference(lat, a, return_scalars=True)
            for f in ("latent_state", "policy_logits", "value", "reward", "value_scalar", "reward_scalar"):
                assert torch.equal(getattr(o, f)[off:off + 8], getattr(ref, f)), (B, off, f)


# ------------------------------------------------------------------------------------------------ tower
@pytest.mark.parametrize("B", (1, 3, 131, 1024))
@pytest.mark.parametrize("kind", ("float", "uint8"))
def test_tower_stages_match_float64(kind, B):
    _, ref64, cu = make_models(A=18, seed=21)
    if kind == "float":
        obs = torch.rand((B,) + OBS, generator=torch.Generator().manual_seed(B)).cuda()
        x64 = obs.double()
    else:
        obs = _atari_frames(B, 4, 64, B).cuda()
        x64 = (obs.double() / 255.0).float().double()
    ds = ref64.representation_network.downsample_net
    raws, infos, vals = [], [], []
    for st in range(9):
        raw, info = dump_stage(cu, obs, st)
        raws.append(raw)
        infos.append(info)
        vals.append(stage_value(raw, info, B))
    inputs = {0: (x64,), 1: (vals[0],), 2: (vals[1],), 3: (vals[1],), 4: (vals[2], vals[3]), 5: (vals[4],), 6: (vals[5],),
              7: (vals[6],)}
    shapes = [32, 32, 16, 16, 16, 16, 8, 8]
    with torch.no_grad():
        for st in range(8):
            y, M, S = stage_reference(ds, st, *inputs[st])
            assert vals[st].shape[-1] == shapes[st] and y.shape == vals[st].shape, (st, y.shape, vals[st].shape)
            r = ((vals[st] - y).abs() / (T_TAU[st] * M + T_ALPHA * S)).max().item()
            assert r <= 1.0, (st, r)
    # stage 8: no pooling2 at 64 px; the fp32 NCHW latent is exactly hi + lo of stage 7, summed in fp32
    assert infos[8][:5] == [64, 8, 8, 0, 0] and infos[8][5] == 1
    g = tcl_grid(raws[7], infos[7], B)[:, 0]
    exp = g[:, 0, :, 1:9, :8].float() + g[:, 1, :, 1:9, :8].float()
    assert torch.equal(raws[8].view(torch.float32).view(B, 64, 8, 8), exp)
    # the latent initial_inference hands on is that tensor through the representation ResBlocks
    assert torch.isfinite(vals[8]).all()


def test_tower_bound_detects_single_pass():
    _, ref64, cu = make_models(A=18, seed=21, math="tc1")
    B = 131
    obs = torch.rand((B,) + OBS, generator=torch.Generator().manual_seed(3)).cuda()
    ds = ref64.representation_network.downsample_net
    vals = [stage_value(*dump_stage(cu, obs, st), B) for st in range(8)]
    inputs = {1: (vals[0],), 2: (vals[1],), 3: (vals[1],), 4: (vals[2], vals[3]), 5: (vals[4],), 7: (vals[6],)}
    with torch.no_grad():
        for st in WGMMA_STAGES:
            y, M, S = stage_reference(ds, st, *inputs[st])
            assert ((vals[st] - y).abs() / (T_TAU[st] * M + T_ALPHA * S)).max().item() > 1.0, st


# ------------------------------------------------------------------------------------------------ searches
SEARCH_CASES = {
    "a6_b1_det_1p": (6, 1, 30, True, "1p"),
    "a6_b131_sto_1p": (6, 131, 40, False, "1p"),
    "a18_b263_det_2p": (18, 263, 30, True, "2p"),
    "a18_b397_sto_mixed": (18, 397, 30, False, "mixed"),
    "a18_b530_sto_2p": (18, 530, 25, False, "2p"),
    "a18_b1201_sto_1p": (18, 1201, 20, False, "1p"),
    "a33_b40_sto_2p": (33, 40, 20, False, "2p"),
}


@pytest.mark.parametrize("name", list(SEARCH_CASES))
def test_fused_search_equals_oracle_driving_the_same_network(name):
    import lightzero_b200 as lzb
    A, B, S, det, players = SEARCH_CASES[name]
    seed = sum(map(ord, name))
    _, _, cu = make_models(A=A, seed=seed % 97)
    latent = make_latents(B, seed)
    legal, logits, noises, tp = search_inputs(B, A, seed, players)
    mcts = lzb.MuZeroMCTSCtree(dict(num_simulations=S, deterministic=det, discount_factor=0.997))
    got, key, plan, roots = fused_search(cu, mcts, S, latent, legal, logits, noises, tp)
    exp, st = oracle_search(cu, S, latent, legal, logits, noises, tp, det, key=key)
    roots.clear()
    if A <= 32:
        R = pick_roots(B)
        assert plan["persistent"] == 1 and plan["R"] == R and plan["ctas"] == -(-B // R), plan
        assert mcts.last_num_kernels == 1
    else:
        assert plan["persistent"] == 0 and mcts.last_num_kernels == 2 * S + 1, plan
    assert_same(got, exp)
    if not det:
        assert st["draws"] > 0, st


def _search_setup(B, A, S, seed, ez=False):
    import lightzero_b200 as lzb
    ref, _, cu = make_models(A=A, seed=seed, ez=ez)
    rng = np.random.default_rng(seed)
    mask = (rng.random((B, A)) < 0.6).astype(np.uint8)
    mask[np.arange(B), rng.integers(0, A, B)] = 1
    legal = [np.nonzero(mask[b])[0].tolist() for b in range(B)]
    noises = [rng.dirichlet([0.3] * len(l)).astype(np.float32).tolist() for l in legal]
    obs = torch.rand((B,) + OBS, generator=torch.Generator().manual_seed(seed))
    if ez:
        mcts = lzb.EfficientZeroMCTSCtree(dict(num_simulations=S, discount_factor=0.997, lstm_horizon_len=5))
    else:
        mcts = lzb.MuZeroMCTSCtree(dict(num_simulations=S, deterministic=True, discount_factor=0.997))
    return cu, obs, mask, legal, noises, mcts


def test_search_with_reuse_equals_stepwise_drive():
    from lightzero_b200 import mz_tree
    from oracle.tree_drive import drive, network, readout
    B, A, S = 96, 6, 30
    cu, obs, mask, legal, noises, mcts = _search_setup(B, A, S, seed=21)
    out = cu.initial_inference(obs.cuda())
    rng = np.random.default_rng(3)
    true_action = [int(l[rng.integers(len(l))]) for l in legal]
    reuse_value = (rng.standard_normal(B) * 0.5).astype(np.float32).tolist()
    roots = mcts.roots(B, legal)
    roots.prepare(0.25, noises, [0.] * B, out.policy_logits, [-1] * B)
    mcts.search_with_reuse(roots, cu, out.latent_state, [-1] * B, true_action, reuse_value)
    fused = readout(roots, A, S)
    roots.clear()
    c = dict(B=B, A=A, S=S, legal=legal, root_logits=out.policy_logits.cpu().numpy(), noises=noises, to_play=[-1] * B,
             true_action=true_action, reuse_value=reuse_value)
    step, _ = drive(mz_tree, c, "reuse", network(cu, out.latent_state))
    assert_same(step, fused)
    counts = step["n_inferred"].tolist()
    assert min(counts) < B


class _EzProxy:
    """not an EfficientZeroModel instance: the mirror drives the device trees one simulation at a time around it"""

    def __init__(self, model):
        self.model = model

    def eval(self):
        return self

    def recurrent_inference(self, latent, hidden, action):
        return self.model.recurrent_inference(latent, hidden, action)


@pytest.mark.parametrize("B,A,S", [(16, 6, 20), (530, 18, 30)])
def test_efficientzero_fused_search_equals_stepwise(B, A, S):
    cu, obs, mask, legal, noises, mcts = _search_setup(B, A, S, seed=B, ez=True)
    out = cu.initial_inference(obs.cuda())
    results = []
    for mode in ("fused", "fused", "step"):
        roots = mcts.roots(B, legal)
        roots.prepare(0.25, noises, [0.] * B, out.policy_logits, [-1] * B)
        mcts.search(roots, cu if mode != "step" else _EzProxy(cu), out.latent_state, out.reward_hidden_state, [-1] * B)
        results.append((roots.get_distributions(), np.asarray(roots.get_values(), np.float32).view(np.uint32).tolist()))
        roots.clear()
    assert results[0] == results[1] == results[2]
    assert all(sum(d) == S for d in results[0][0])


@pytest.mark.parametrize("hc", [16, 8])
def test_efficientzero_trunk_features_and_lstm(hc):
    """hc = 16: nin = 1024, hc = 8: nin = 512 (both k_ez_lstm_tc); lstm_hidden_size 48 is not a multiple of 64 (k_ez_lstm)"""
    import lightzero_b200 as lzb
    from oracle.model_ref import EfficientZeroModelRef, emulate_trained_
    A, B = 6, 397
    for H in (512, 48):
        torch.manual_seed(40 + hc)
        kw = dict(reward_head_channels=hc, lstm_hidden_size=H)
        ref = emulate_trained_(EfficientZeroModelRef(OBS, A, **kw), 40 + hc)
        cu = lzb.EfficientZeroModel(observation_shape=OBS, action_space_size=A, downsample=True, **kw).load_state_dict(ref.state_dict())
        ref64 = copy.deepcopy(ref).double().cuda().eval()
        latent, action = make_latents(B, seed=hc, peak=3.0), (torch.arange(B) % A).cuda()
        for which in (0, 1):
            ratios, out, _ = run_program(cu, ref64, which, latent, action)
            assert max(ratios.values()) <= 1.0, ratios
            if which == 0:
                assert out["feat"].shape == (B, hc * P)
                feat = out["feat"].double()
            check_scalars(out, which, True)
        g = torch.Generator().manual_seed(hc)
        h0, c0 = (0.5 * torch.randn(B, H, generator=g)).cuda(), (2.0 * torch.randn(B, H, generator=g)).cuda()
        o = cu.recurrent_inference(latent, (h0[None], c0[None]), action)
        with torch.no_grad():
            h1, c1, eh, ec = lstm_bound(ref64.dynamics_network.lstm, feat, h0.double(), c0.double())
        nh, nc = o.reward_hidden_state
        assert worst(nh[0].double() - h1, eh) <= 1.0 and worst(nc[0].double() - c1, ec) <= 1.0


def test_uint8_frames_equal_scaled_float_frames_bit_for_bit():
    from lightzero_b200.collect import MuZeroCollectPolicy
    B, A, S = 48, 6, 12
    cu, obs, mask, legal, noises, mcts = _search_setup(B, A, S, seed=5)
    u8 = torch.randint(0, 256, (B,) + OBS, dtype=torch.uint8, generator=torch.Generator().manual_seed(3))
    f32 = torch.from_numpy((u8.numpy() / 255.).astype(np.float32))
    pol = MuZeroCollectPolicy(cu, dict(num_simulations=S, deterministic=True, discount_factor=0.997))
    noise = np.zeros((B, A), np.float32)
    for b in range(B):
        noise[b, :len(noises[b])] = noises[b]
    res = []
    for o in (f32.pin_memory(), u8.pin_memory(), u8.cuda(), f32.cuda()):
        r = pol.search_batch(o, torch.from_numpy(mask), torch.from_numpy(noise), None, deterministic=True, read_back=True)
        res.append({k: v.clone() for k, v in r.items()})
    for r in res[1:]:
        for k in ("visits", "values", "pred_value", "policy_logits"):
            a, b = res[0][k], r[k]
            assert torch.equal(a.view(torch.int32) if a.dtype == torch.float32 else a, b.view(torch.int32) if b.dtype == torch.float32 else b), k


def test_frame_stack_collect_equals_float_frames():
    """FrameStack-style uint8 stacks through lz_search_collect_u8 == the same stacks scaled to float32 on the host"""
    from lightzero_b200.collect import MuZeroCollectPolicy
    B, A, S = 24, 18, 10
    cu, obs, mask, legal, noises, mcts = _search_setup(B, A, S, seed=8)
    frames = _atari_frames(B + 3, 1, 64, 4)[:, 0]
    u8 = torch.stack([frames[b:b + 4] for b in range(B)])          # overlapping 4-frame stacks
    f32 = (u8.double() / 255.0).float()
    pol = MuZeroCollectPolicy(cu, dict(num_simulations=S, deterministic=True, discount_factor=0.997))
    noise = torch.zeros(B, A)
    a = pol.search_batch(u8.cuda(), torch.from_numpy(mask), noise, None, deterministic=True, read_back=True)
    a = {k: v.clone() for k, v in a.items()}
    b = pol.search_batch(f32.cuda(), torch.from_numpy(mask), noise, None, deterministic=True, read_back=True)
    for k in ("visits", "values", "pred_value", "policy_logits"):
        x, y = a[k], b[k]
        assert torch.equal(x.view(torch.int32) if x.dtype == torch.float32 else x, y.view(torch.int32) if y.dtype == torch.float32 else y), k


def test_refusals():
    import lightzero_b200 as lzb
    _, _, cu = make_models(A=6, seed=1)
    with pytest.raises(Exception, match="tc3"):
        cu.set_math("fp32")
    cu.set_math("tc1")
    cu.set_math("tc3")
    for px in (32, 72, 128):
        with pytest.raises(Exception, match="not supported"):
            lzb.MuZeroModel(observation_shape=(4, px, px), action_space_size=6, downsample=True)
    # the reference's default downsample=False builds a full-resolution 64x64 network: not implemented here, so a 64x64
    # model must ask for DownSample as the shipped Atari configs do; 84 / 96 keep their DownSample default
    for cls in (lzb.MuZeroModel, lzb.EfficientZeroModel):
        for kw in ({}, dict(downsample=False)):
            with pytest.raises(NotImplementedError, match="downsample"):
                cls(observation_shape=(4, 64, 64), action_space_size=6, **kw)
        assert cls(observation_shape=(4, 64, 64), action_space_size=6, downsample=True).latent_hw == 8
        assert cls(observation_shape=(4, 96, 96), action_space_size=6).latent_hw == 6
