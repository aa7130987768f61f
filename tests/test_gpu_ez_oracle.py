"""The EfficientZero value-prefix path against float64, and the fused EfficientZero search against the oracle driving the
same network, bit for bit.

Part 1: one LSTM step (k_ez_lstm_tc, 3xFP16 wgmma, or the fp32 k_ez_lstm) and the value-prefix head (k_ez_head:
BatchNorm1d -> ReLU -> Linear(H, hid) -> BN -> ReLU -> Linear(hid, K) -> softmax expectation -> h^-1) over a table of
latent grids, LSTM sizes, head sizes and supports.  The LSTM's h' / c' are held to ``lstm_bound`` on the kernel's own
reward features (lz_model_debug_net_stage); the value-prefix logits to a float64 head on the kernel's own h' (with no
reset, reward_hidden_state[0] is the h' k_ez_head reads) under |y - y64| <= TAU_HEAD * M + ALPHA, M carried through
|BN|, |W1|, |W2| as head_reference does; the scalars to h^-1 of the kernel's own logits within the 2e-4 quantum
(DESIGN.md 4.4).  Both bounds are tighter than test_gpu_net_layers.py's LSTM bound so that a lost pass cannot hide: in
float64, dropping the lo parts of W_ih / W_hh exceeds the LSTM bound by >= 8x and TF32-rounded FC weights exceed the head
bound by >= 8x.  TAU_LSTM and TAU_HEAD are calibrated on an H100 (DESIGN.md 4.5).

Part 2: ``oracle_search_ez`` is the reference loop (mcts_ctree.py:729-876) on oracle.ctree_port_ez with the CUDA network
evaluating the leaves: latents and (h, c) gathered from pools at the oracle's (ix, iy), ``recurrent_inference(...,
return_scalars=True)``, is_reset = search_len % lstm_horizon_len == 0, the stored h / c of reset leaves zeroed, and the
kernel's own value_prefix_scalar / value_scalar / logits backed up.  The fused ``EfficientZeroMCTSCtree.search`` on the
same roots, noise and to_play must give the same visit counts, root-value bits and trajectories.  This rests on a root's
outputs not depending on its row in the LSTM tile or the head CTA, which ``test_root_outputs_identical_at_every_row``
checks directly.  Every search case asserts the branch it is named for from the oracle's counters and prints them.
"""
import copy
import re
import time

import numpy as np
import pytest
import torch

from test_gpu_net_layers import ALPHA, _bn, inverse_h, lstm_bound, make_latents as latents6, net_stage as net_stage6, \
    pow2_hi, program, split_full, worst
from test_gpu_obs64 import make_latents as latents8, net_stage as net_stage8
from oracle.tree_drive import assert_same, drive, network, readout
from test_gpu_search_oracle import _inputs, _prepare, debug_rng, differ, near_policy, peaked_zero_values, visits_sum_to, \
    zero_policy

pytestmark = pytest.mark.gpu

SUPPORTS = {21: (-10., 11., 1.), 101: (-50., 51., 1.), 601: (-300., 301., 1.), 608: (-304., 304., 1.)}
# calibrated on an H100 (DESIGN.md 4.5): the kernels stay under a quarter of each bound, and a dropped lo pass of the
# LSTM weights or TF32 FC weights in the head exceed it by >= 8x
TAU_LSTM = 2.0 ** -19
TAU_HEAD = 2.0 ** -22


# ------------------------------------------------------------------------------------------------ models and inputs
def make_ez(obs, A, hc, H, hid, K, seed, mutate=None):
    """(float64 reference on the GPU, CUDA EfficientZeroModel); obs 96 -> 6x6 latent grid, 64 -> 8x8"""
    import lightzero_b200 as lzb
    from oracle.model_ref import EfficientZeroModelRef, emulate_trained_
    torch.manual_seed(seed)
    sup = SUPPORTS[K]
    kw = dict(num_res_blocks=1, reward_head_channels=hc, lstm_hidden_size=H, reward_head_hidden_channels=(hid,),
              reward_support_range=sup, value_support_range=sup)
    shape = (4, obs, obs)
    ref = emulate_trained_(EfficientZeroModelRef(shape, A, **kw), seed)
    if mutate is not None:
        mutate(ref)
    cu = lzb.EfficientZeroModel(observation_shape=shape, action_space_size=A, downsample=True, **kw).load_state_dict(ref.state_dict())
    return copy.deepcopy(ref).double().cuda().eval(), cu


def lstm_kernel(obs, hc, H):
    """the LSTM kernel ez_launch picks (test_lstm_kernel_by_name checks it on the device)"""
    nin = hc * (36 if obs == 96 else 64)
    return "k_ez_lstm_tc" if nin % 64 == 0 and H % 64 == 0 else "k_ez_lstm"


def latents(cu, B, seed):
    """post-ReLU latents with the batch maximum at 3 (the LSTM gates then span the sigmoid), root 0 all zero"""
    x = (latents6 if cu.latent_hw == 6 else latents8)(B, seed, peak=3.0)
    x[0] = 0.0
    return x


def hidden(B, H, seed):
    """h0 in (-1, 1); c0 ~ 3 N(0, 1), through the linear and the saturated part of tanh; the last root has h0 = c0 = 0
    (the state after initial_inference)"""
    g = torch.Generator().manual_seed(seed)
    h0, c0 = 2.0 * torch.rand(B, H, generator=g) - 1.0, 3.0 * torch.randn(B, H, generator=g)
    h0[-1], c0[-1] = 0.0, 0.0
    return h0.cuda(), c0.cuda()


def features(cu, ref64, latent, action):
    """the kernel's own reward features [B][hc * P] (the LSTM input) from the recurrent program's hook"""
    nl = len(program(ref64, 0)[0])
    buf, _ = (net_stage6 if cu.latent_hw == 6 else net_stage8)(cu, 0, latent, action, nl, nl)
    nfeat = cu._cfg.reward_head_channels * cu.latent_hw ** 2
    return split_full(buf, latent.shape[0], cu.value_support_size, cu.action_space_size, nfeat)["feat"].double()


def tf32(w):
    """w rounded to TF32 (10 mantissa bits, nearest, ties away from zero)"""
    i = w.float().view(torch.int32)
    return ((i + 0x1000) & -0x2000).view(torch.float32).double()


def vp_head(dyn, h, round_fc=None):
    """(logits, M) of norm_value_prefix -> ReLU -> fc_reward_head on h' in float64; round_fc rounds W1 and W2"""
    lin1, bn1, lin2 = dyn.fc_reward_head[0], dyn.fc_reward_head[1], dyn.fc_reward_head[3]
    W1, W2 = lin1.weight, lin2.weight
    if round_fc is not None:
        W1, W2 = round_fc(W1), round_fc(W2)
    s0, m0, b0 = _bn(dyn.norm_value_prefix, (1, -1))
    x, Mx = torch.relu(s0 * (h - m0) + b0), s0.abs() * (h.abs() + m0.abs()) + b0.abs()
    u, Mu = x @ W1.T + lin1.bias, Mx @ W1.abs().T + lin1.bias.abs()
    s1, m1, b1 = _bn(bn1, (1, -1))
    g, Mg = torch.relu(s1 * (u - m1) + b1), s1.abs() * (Mu + m1.abs()) + b1.abs()
    return g @ W2.T + lin2.bias, Mg @ W2.abs().T + lin2.bias.abs()


def check_batch(cu, ref64, K, B, seed, sensitivity=False):
    """one recurrent_inference of B roots against float64: {name: worst |err| / bound}; scalars asserted"""
    A, H = cu.action_space_size, cu.lstm_hidden_size
    latent, action = latents(cu, B, seed), (torch.arange(B) % A).cuda()
    h0, c0 = hidden(B, H, seed)
    feat = features(cu, ref64, latent, action)
    o = cu.recurrent_inference(latent, (h0[None], c0[None]), action, return_scalars=True)
    dyn = ref64.dynamics_network
    nh, nc = o.reward_hidden_state[0][0].double(), o.reward_hidden_state[1][0].double()
    r = {}
    with torch.no_grad():
        h1, c1, eh, ec = lstm_bound(dyn.lstm, feat, h0.double(), c0.double(), tau=TAU_LSTM)
        r["h"], r["c"] = worst(nh - h1, eh), worst(nc - c1, ec)
        y, M = vp_head(dyn, nh)
        err = o.value_prefix.double() - y
        r["head"], r["head_err/M"] = worst(err, TAU_HEAD * M + ALPHA), worst(err, M)
        if sensitivity:
            Wi, Wh = dyn.lstm.weight_ih_l0, dyn.lstm.weight_hh_l0
            Wc = pow2_hi(torch.cat([Wi, Wh], 1))          # one power-of-two scale over both, as ez_pack_wtc packs them
            h2, c2, _, _ = lstm_bound(dyn.lstm, feat, h0.double(), c0.double(), tau=TAU_LSTM,
                                      weights=(Wc[:, :Wi.shape[1]], Wc[:, Wi.shape[1]:]))
            r["hi-only h"], r["hi-only c"] = worst(h2 - h1, eh), worst(c2 - c1, ec)
            r["tf32 head"] = worst(vp_head(dyn, nh, tf32)[0] - y, TAU_HEAD * M + ALPHA)
    sup = SUPPORTS[K]
    for name, got, logits in (("value_prefix", o.value_prefix_scalar, o.value_prefix), ("value", o.value_scalar, o.value)):
        exp = inverse_h(logits, sup)
        assert torch.isfinite(got).all(), name
        bad = (got.double() - exp).abs() > 2e-4 * torch.clamp(exp.abs(), min=1.0)
        assert not bad.any(), (name, B, int(bad.sum()), (got.double() - exp).abs().max().item())
    return r


# ------------------------------------------------------------------------------------------------ configurations
# (observation px, A, reward-head channels hc, lstm_hidden_size H, reward-head hidden hid, support size K)
CONFIGS = [
    (96, 6, 16, 512, 32, 601),      # the 96x96 default: nin 576, 17 chunks (odd)
    (96, 9, 16, 64, 8, 101),        # H = 64: 4 column tiles, 10 chunks
    (96, 6, 8, 512, 8, 608),        # nin 288: k_ez_lstm, K = 608 (the largest head)
    (96, 6, 1, 16, 1, 21),          # nin 36: nin + H = 52 is not a multiple of k_ez_lstm's 16-wide k-tile
    (96, 6, 1, 48, 32, 601),
    (64, 18, 16, 512, 32, 101),     # the shipped Atari EfficientZero config (atari_efficientzero_config.py): 24 chunks (even)
    (64, 6, 1, 64, 8, 21),          # nin + H = 128: 2 chunks, fewer than the 3 ring stages
    (64, 6, 1, 128, 32, 608),       # 3 chunks, as many as the ring stages
    (64, 6, 16, 256, 1, 601),       # 20 chunks
    (64, 6, 8, 48, 1, 101),         # H = 48: k_ez_lstm on the 8x8 grid
]
ATARI = (64, 18, 16, 512, 32, 101)


def _cfg_id(c):
    return f"px{c[0]}-A{c[1]}-hc{c[2]}-H{c[3]}-hid{c[4]}-K{c[5]}"


def _chunks(c):
    return (c[2] * (36 if c[0] == 96 else 64) + c[3]) // 64


def test_configurations_cover_every_value():
    assert {(c[0], lstm_kernel(c[0], c[2], c[3])) for c in CONFIGS} == \
        {(px, k) for px in (96, 64) for k in ("k_ez_lstm_tc", "k_ez_lstm")}
    chunks = {_chunks(c) for c in CONFIGS if lstm_kernel(c[0], c[2], c[3]) == "k_ez_lstm_tc"}
    assert {2, 3, 17, 24} <= chunks
    assert {c[3] for c in CONFIGS} >= {16, 48, 64, 128, 256, 512}
    assert {c[4] for c in CONFIGS} == {1, 8, 32}
    assert {c[5] for c in CONFIGS} == {21, 101, 601, 608}
    assert {c[2] for c in CONFIGS} == {1, 8, 16}
    assert any(c[0] == 96 and c[2] == 1 and (36 + c[3]) % 16 for c in CONFIGS)
    assert ATARI in CONFIGS
    assert all(len(np.arange(*SUPPORTS[K])) == K for K in SUPPORTS)


@pytest.mark.parametrize("cfg", CONFIGS, ids=[_cfg_id(c) for c in CONFIGS])
def test_lstm_and_value_prefix_head_match_float64(cfg):
    obs, A, hc, H, hid, K = cfg
    ref64, cu = make_ez(obs, A, hc, H, hid, K, seed=A + hc + H)
    assert cu.latent_hw == (6 if obs == 96 else 8)
    for B in (1, 129, 397):
        r = check_batch(cu, ref64, K, B, seed=B + H, sensitivity=B == 397)
        print(f"\n[ez-f64] {_cfg_id(cfg)} {lstm_kernel(obs, hc, H)} B={B}: " + " ".join(f"{k}={v:.3g}" for k, v in r.items()))
        over = {k: v for k, v in r.items() if k in ("h", "c", "head") and not v <= 1.0}
        assert not over, f"{_cfg_id(cfg)} B={B}: over the float64 bound: {over}"
        if B == 397:
            weak = {k: v for k, v in r.items() if k in ("hi-only h", "hi-only c", "tf32 head") and not v >= 8.0}
            assert not weak, f"{_cfg_id(cfg)}: a lost pass would stay within 8x of the bound: {weak}"


def _kernels(fn):
    """names of the k_ez_* kernels a call launches (torch.profiler, CUDA activities)"""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return {m for e in prof.events() for m in re.findall(r"k_ez_\w+", e.name)}


def test_lstm_kernel_by_name():
    """the kernel that ran, by name, for every configuration (the search cases report lstm_kernel from this rule)"""
    for obs, A, hc, H, hid, K in CONFIGS:
        _, cu = make_ez(obs, A, hc, H, hid, K, seed=1)
        B = 5
        latent, action = latents(cu, B, 1), (torch.arange(B) % A).cuda()
        h0, c0 = hidden(B, H, 1)
        ran = _kernels(lambda: cu.recurrent_inference(latent, (h0[None], c0[None]), action, return_scalars=True))
        assert ran == {lstm_kernel(obs, hc, H), "k_ez_head"}, (obs, hc, H, ran)


EDGE_B = (1, 2, 3, 63, 64, 65, 127, 128, 129, 255, 257, 1024, 1201)


@pytest.mark.parametrize("cfg", [ATARI, (96, 6, 8, 512, 8, 608)], ids=["k_ez_lstm_tc", "k_ez_lstm"])
def test_batch_edges_match_float64(cfg):
    """the 64-row fp32 tile, the 128-row tensor-core tile and the 2-root head CTA, with partial last tiles"""
    obs, A, hc, H, hid, K = cfg
    ref64, cu = make_ez(obs, A, hc, H, hid, K, seed=7)
    worst_r = {}
    for B in EDGE_B:
        r = check_batch(cu, ref64, K, B, seed=B)
        for k in ("h", "c", "head"):
            worst_r[k] = max(worst_r.get(k, 0.0), r[k])
        assert max(r["h"], r["c"], r["head"]) <= 1.0, (B, r)
    print(f"\n[ez-f64] batch edges {_cfg_id(cfg)}: " + " ".join(f"{k}={v:.3g}" for k, v in worst_r.items()))


@pytest.mark.parametrize("cfg", [ATARI, (96, 6, 8, 512, 8, 608)], ids=["k_ez_lstm_tc", "k_ez_lstm"])
def test_root_outputs_identical_at_every_row(cfg):
    """One root's h', c', value-prefix logits and both scalars are the same bits alone, at every row of an LSTM tile
    (position p = 129 i sits at row i of its 128-row tile, and at every row of a 64-row tile and of a 2-root head CTA), and
    with or without return_scalars."""
    obs, A, hc, H, hid, K = cfg
    _, cu = make_ez(obs, A, hc, H, hid, K, seed=9)
    t_lat, t_act = latents(cu, 2, 3)[1:2], torch.tensor([A - 1]).cuda()
    g = torch.Generator().manual_seed(4)
    t_h, t_c = (2.0 * torch.rand(1, H, generator=g) - 1.0).cuda(), (3.0 * torch.randn(1, H, generator=g)).cuda()

    def run(lat, h, c, act, rs):
        o = cu.recurrent_inference(lat, (h[None], c[None]), act, return_scalars=rs)
        out = dict(h=o.reward_hidden_state[0][0], c=o.reward_hidden_state[1][0], vp=o.value_prefix)
        if rs:
            out.update(vps=o.value_prefix_scalar, vs=o.value_scalar)
        return out

    alone = run(t_lat, t_h, t_c, t_act, True)
    pos = [129 * i for i in range(128)]
    B = pos[-1] + 2
    lat, act = latents(cu, B, 5), (torch.arange(B) % A).cuda()
    h, c = hidden(B, H, 6)
    lat[pos], act[pos], h[pos], c[pos] = t_lat, t_act, t_h, t_c
    assert {p % 128 for p in pos} == set(range(128)) and {p % 2 for p in pos} == {0, 1}
    for rs in (True, False):
        got = run(lat, h, c, act, rs)
        for k, v in got.items():
            same = (v[pos].view(torch.int32) == alone[k][0].view(torch.int32)).reshape(len(pos), -1).all(1)
            assert same.all(), (rs, k, [p for p, s in zip(pos, same.tolist()) if not s][:8])


# ------------------------------------------------------------------------------------------------ the two searches
def fused_search_ez(cu, mcts, latent, h0, c0, legal, logits, noises, tp, cap=None, roots=None):
    """EfficientZeroMCTSCtree.search; `cap`: tree capacity (max_sims) larger than S"""
    if roots is None:
        roots = mcts.roots(len(tp), legal)
    _prepare(roots, logits, noises, tp)
    if cap is not None:
        roots._materialize(cap)
    mcts.search(roots, cu, latent, (h0[None], c0[None]), tp)
    return readout(roots, logits.shape[1], int(mcts._cfg.num_simulations)), debug_rng(roots), roots


def oracle_search_ez(cu, S, horizon, latent, h0, c0, legal, logits, noises, tp, det, key=None, step0=0, discount=0.997,
                     delta=0.01, zero_reset_state=True, reset_in_backup=True):
    """The reference loop (mcts_ctree.py:729-876, oracle/tree_drive.py) on oracle.ctree_port_ez with the CUDA network
    evaluating the leaves.  Returns (trace, tie statistics, resets)."""
    from oracle import ctree_port_ez as port
    c = dict(B=len(tp), A=logits.shape[1], S=S, legal=legal, root_logits=logits, noises=noises, to_play=tp,
             discount=discount, delta=delta, lstm_horizon_len=horizon)
    setup = None if det else (lambda r: r.set_tie_hash(key[0], key[1], step0))
    trace, roots = drive(port, c, "ez", network(cu, latent, (h0, c0), zero_reset_state), setup=setup,
                         reset_in_backup=reset_in_backup)
    return trace, roots.tie_stats(), int(trace["is_reset"].sum())


def _setup(spec, A, B, seed, players, ikw, mutate=None, zero_hidden=False):
    obs, hc, H, hid, K = spec
    _, cu = make_ez(obs, A, hc, H, hid, K, seed=seed % 97, mutate=mutate)
    latent = latents(cu, B, seed)
    h0, c0 = hidden(B, H, seed)
    if zero_hidden:
        h0, c0 = torch.zeros_like(h0), torch.zeros_like(c0)
    legal, logits, noises, tp = _inputs(B, A, seed, players, **ikw)
    return cu, latent, h0, c0, legal, logits, noises, tp


def _mcts(S, det, horizon, **kw):
    import lightzero_b200 as lzb
    return lzb.EfficientZeroMCTSCtree(dict(dict(num_simulations=S, deterministic=det, discount_factor=0.997,
                                                lstm_horizon_len=horizon), **kw))


def _report(name, st, resets, kernel, nk, seconds):
    print(f"\n[ez-search-oracle] {name}: resets={resets} ties={st['ties']} draws={st['draws']} near={st['near']} "
          f"max_len={st['max_len']} lstm={kernel} kernels={nk} {seconds:.1f}s")


# ------------------------------------------------------------------------------------------------ the case matrix
D96 = (96, 16, 512, 32, 601)            # the 96x96 default (k_ez_lstm_tc, 17 chunks)
ATARI_SPEC = (64, 16, 512, 32, 101)     # atari_efficientzero_config.py (k_ez_lstm_tc, 24 chunks)
# name: model (px, hc, H, hid, K), A, B, S, horizon, deterministic, players, model mutation, input kwargs, tree capacity,
# zero root hidden state
CASES = {
    "atari_a18_b1024_s50_h5_det": (ATARI_SPEC, 18, 1024, 50, 5, True, "1p", None, {}, None, True),
    "atari_a18_b1024_s50_h5_sto": (ATARI_SPEC, 18, 1024, 50, 5, False, "1p", None, {}, None, True),
    "d96_a6_b256_s40_h3_sto_2p": (D96, 6, 256, 40, 3, False, "2p", None, {}, None, False),
    "d96_a33_b1201_s20_h2_sto_mixed": (D96, 33, 1201, 20, 2, False, "mixed", None, {}, None, False),
    "fp32_hc8_px96_a9_b300_s30_h3_sto_2p": ((96, 8, 512, 32, 601), 9, 300, 30, 3, False, "2p", None, {}, None, False),
    "fp32_H48_px64_a6_b200_s30_h4_sto_mixed": ((64, 16, 48, 32, 101), 6, 200, 30, 4, False, "mixed", None, {}, None, False),
    "a1_b3_s200_h5_sto": (D96, 1, 3, 200, 5, False, "1p", None, dict(masks=False), None, False),
    "a2_b7_s133_h5_sto_peaked_cap256": (D96, 2, 7, 133, 5, False, "1p", peaked_zero_values, dict(noise=False), 256, False),
    "h1_2chunk_a6_b64_s30_sto": ((64, 1, 64, 8, 21), 6, 64, 30, 1, False, "1p", None, {}, None, False),
    "h25_3chunk_a6_b64_s20_sto": ((64, 1, 128, 32, 608), 6, 64, 20, 25, False, "2p", None, {}, None, False),
    "a6_b1_s1_sto": (D96, 6, 1, 1, 5, False, "1p", None, dict(noise=False, tie_root=True), None, False),
    "a31_b300_s30_h3_sto_zero_policy": (D96, 31, 300, 30, 3, False, "1p", zero_policy, dict(noise=False, tie_root=True), None, False),
    "a32_b531_s30_h4_sto_2p_near_ties": (D96, 32, 531, 30, 4, False, "2p", near_policy, dict(noise=False), None, False),
    "a32_b531_s30_h2_det_zero_policy": (D96, 32, 531, 30, 2, True, "mixed", zero_policy, dict(noise=False, tie_root=True), None, False),
}


@pytest.mark.parametrize("name", list(CASES))
def test_fused_ez_search_equals_oracle_driving_the_same_network(name):
    spec, A, B, S, horizon, det, players, mutate, ikw, cap, zero_hidden = CASES[name]
    t0 = time.time()
    seed = sum(map(ord, name))
    cu, latent, h0, c0, legal, logits, noises, tp = _setup(spec, A, B, seed, players, ikw, mutate, zero_hidden)
    mcts = _mcts(S, det, horizon)
    got, key, roots = fused_search_ez(cu, mcts, latent, h0, c0, legal, logits, noises, tp, cap=cap)
    exp, st, resets = oracle_search_ez(cu, S, horizon, latent, h0, c0, legal, logits, noises, tp, det, key=key)
    nk = mcts.last_num_kernels
    roots.clear()
    kernel = lstm_kernel(spec[0], spec[1], spec[2])
    _report(name, st, resets, kernel, nk, time.time() - t0)
    assert_same(got, exp)
    assert visits_sum_to(got, S)
    assert nk == 1 + 4 * S
    # the branch the case is named for
    assert _kernels(lambda: cu.recurrent_inference(latent[:1], (h0[:1][None], c0[:1][None]), torch.zeros(1, dtype=torch.long).cuda())) \
        == {kernel, "k_ez_head"}
    if name.startswith("fp32"):
        assert kernel == "k_ez_lstm"
    if "chunk" in name or name.startswith(("atari", "d96")):
        assert kernel == "k_ez_lstm_tc"
    if not det and S > 1 and A > 1:
        assert st["ties"] > 0 and st["draws"] > 0
    if horizon == 1:
        assert resets == B * S                 # every leaf resets
    elif horizon > S:
        assert resets == 0
    elif S > 1:
        assert resets > 0
    if "2p" in name or "mixed" in name:
        assert len(set(tp)) > 1
    if "near" in name:
        assert st["near"] > 0
    if "zero_policy" in name:
        assert st["ties"] >= B * S // 4
    if name.startswith("a1_"):
        assert st["max_len"] == S and resets == B * (S // horizon)
    if "peaked" in name:
        assert st["max_len"] >= 64 and resets >= B * 10
    if S == 1:
        assert st["max_len"] == 1


def test_discount_and_value_delta_max():
    """non-default discount and MinMax value_delta_max in the EfficientZero back-up"""
    A, B, S, H = 9, 96, 40, 3
    cu, latent, h0, c0, legal, logits, noises, tp = _setup(D96, A, B, 31, "2p", {})
    mcts = _mcts(S, False, H, discount_factor=0.9, value_delta_max=0.05)
    got, key, roots = fused_search_ez(cu, mcts, latent, h0, c0, legal, logits, noises, tp)
    roots.clear()
    exp, st, resets = oracle_search_ez(cu, S, H, latent, h0, c0, legal, logits, noises, tp, False, key=key, discount=0.9, delta=0.05)
    default, _, _ = oracle_search_ez(cu, S, H, latent, h0, c0, legal, logits, noises, tp, False, key=key)
    _report("a9_b96_s40_h3_sto_2p_discount0.9_delta0.05", st, resets, lstm_kernel(96, 16, 512), mcts.last_num_kernels, 0.0)
    assert_same(got, exp)
    assert not np.array_equal(got["distributions"], default["distributions"])
    assert st["draws"] > 0 and resets > 0


def test_repeated_stochastic_searches_on_one_pooled_tree():
    """Two stochastic searches on the same tree: the second runs at the next epoch, must match the oracle there and must
    differ from the first."""
    A, B, S, H = 18, 200, 30, 4
    cu, latent, h0, c0, legal, logits, noises, tp = _setup(D96, A, B, 41, "1p", dict(noise=False, tie_root=True), zero_policy)
    mcts = _mcts(S, False, H)
    roots = mcts.roots(B, legal)
    first, key1, roots = fused_search_ez(cu, mcts, latent, h0, c0, legal, logits, noises, tp, roots=roots)
    handle = roots._tree
    second, key2, roots = fused_search_ez(cu, mcts, latent, h0, c0, legal, logits, noises, tp, roots=roots)
    assert roots._tree is handle and key2[0] == key1[0] and key2[1] > key1[1]     # every reset advances the epoch
    roots.clear()
    for got, key in ((first, key1), (second, key2)):
        exp, st, resets = oracle_search_ez(cu, S, H, latent, h0, c0, legal, logits, noises, tp, False, key=key)
        assert_same(got, exp)
    _report("a18_b200_s30_h4_sto_repeated", st, resets, lstm_kernel(96, 16, 512), mcts.last_num_kernels, 0.0)
    assert not np.array_equal(first["distributions"], second["distributions"]) and st["draws"] > 0 and resets > 0


def test_sensitivity_of_the_comparison():
    """Oracle mutations the comparison must catch on reset- and tie-rich roots (the device is unchanged): the horizon
    +- 1, the stored state of reset leaves not zeroed, is_reset withheld from the back-up, the wrong epoch and the wrong
    step.  Each must disagree with the device on most roots."""
    A, B, S, H = 4, 132, 30, 2
    cu, latent, h0, c0, legal, logits, noises, tp = _setup(D96, A, B, 51, "1p", dict(noise=False, tie_root=True), zero_policy)
    mcts = _mcts(S, False, H)
    got, key, roots = fused_search_ez(cu, mcts, latent, h0, c0, legal, logits, noises, tp)
    roots.clear()
    run = lambda **kw: oracle_search_ez(cu, S, kw.pop("horizon", H), latent, h0, c0, legal, logits, noises, tp, False,
                                        **dict(dict(key=key), **kw))
    exp, st, resets = run()
    assert_same(got, exp)
    assert resets >= B * S // 4 and st["draws"] > 0

    def frac(o):
        return float(differ(got, o[0]).mean())
    fr = {
        "horizon-1": frac(run(horizon=H - 1)),
        "horizon+1": frac(run(horizon=H + 1)),
        "state not zeroed at reset": frac(run(zero_reset_state=False)),
        "is_reset withheld from the back-up": frac(run(reset_in_backup=False)),
        "epoch+1": frac(run(key=(key[0], key[1] + 1))),
        "step+1": frac(run(step0=1)),
    }
    print(f"\n[ez-search-oracle] sensitivity ({B} roots, resets={resets}, draws={st['draws']}), fraction of roots that "
          "disagree: " + ", ".join(f"{k} {v:.3f}" for k, v in fr.items()))
    assert min(fr.values()) > 0.5, fr
