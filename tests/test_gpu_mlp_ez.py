"""GPU tests of EfficientZeroModelMLP (csrc/mlp_tc.cu + the value-prefix head of ez.cu):
- the CUDA model against the reference class's fixtures and the PyTorch restatement, both programs, at B from 1 to 1201
  (partial last CTAs included): 1e-5 on latents, logits and the LSTM state, 2e-4 on scalars;
- one root gives the same bits at every slot and packing;
- the fused EfficientZero searches (search, search_with_reuse), collect and reanalyze against the oracle driving the same
  network, bit for bit;
- the refusals of the accepted space."""
import numpy as np
import pytest
import torch

import mlp_ez_model_ref as MR
from conftest import ROOT
from oracle.tree_drive import assert_same, drive, network, readout
from test_gpu_search_oracle import _inputs, _prepare, debug_rng, visits_sum_to

pytestmark = pytest.mark.gpu

NAMES = list(MR.CONFIGS)
BATCHES = (1, 2, 3, 63, 64, 65, 127, 128, 129, 1024, 1201)


def make(name, seed=0, math="tc3", ssl_keys=True):
    """(restatement on the CPU, CUDA model loaded from its state_dict); the SSL heads' keys ride along and are ignored"""
    import lightzero_b200 as lzb
    ref = MR.build(name, seed)
    sd = dict(ref.state_dict())
    if ssl_keys:
        sd["projection.0.weight"] = torch.randn(8, 8)
        sd["prediction_head.0.weight"] = torch.randn(8, 8)
    cu = lzb.EfficientZeroModelMLP(**MR.model_kwargs(name)).load_state_dict(sd)
    cu.set_math(math)
    return ref, cu


@torch.no_grad()
def zero_policy(ref):
    """policy FC2 weights and bias zero: every prior is uniform, unvisited siblings tie exactly"""
    fc = ref.prediction_network.fc_policy_head[-1]
    fc.weight.zero_()
    fc.bias.zero_()


def scalar(logits):
    """softmax . support -> h^-1 in float64 (support (-300, 301, 1))"""
    x = torch.as_tensor(logits).double()
    v = (torch.softmax(x, -1) * torch.arange(-300, 301, dtype=torch.float64)).sum(-1)
    eps = 0.001
    return torch.sign(v) * (((torch.sqrt(1 + 4 * eps * (torch.abs(v) + 1 + eps)) - 1) / (2 * eps)) ** 2 - 1)


def close(got, exp, what, atol=1e-5, rtol=1e-5):
    got, exp = torch.as_tensor(got).double().cpu(), torch.as_tensor(exp).double().cpu()
    err = ((got - exp).abs() - rtol * exp.abs()).max().item()
    assert err <= atol, f"{what}: max excess error {err:.3g}"


def inputs(name, B, seed):
    obs_dim, A, L, H, _ = MR.CONFIGS[name]
    g = torch.Generator().manual_seed(seed)
    obs = torch.rand((B, obs_dim), generator=g) * 2.0 - 1.0
    action = torch.randint(0, A, (B,), generator=g)
    h0 = (torch.rand((1, B, H), generator=g) * 2.0 - 1.0) * 0.5
    c0 = torch.randn((1, B, H), generator=g)
    return obs, action, h0, c0


def run_both(ref, cu, obs, action, h0, c0):
    with torch.no_grad():
        r0 = ref.initial_inference(obs)
        r1 = ref.recurrent_inference(r0.latent_state, (h0, c0), action)
    g0 = cu.initial_inference(obs.cuda(), return_scalar_value=True)
    g1 = cu.recurrent_inference(r0.latent_state.cuda(), (h0.cuda(), c0.cuda()), action.cuda(), return_scalars=True)
    return r0, r1, g0, g1


def check(r0, r1, g0, g1, tag):
    close(g0.latent_state, r0.latent_state, f"{tag} init latent")
    close(g0.policy_logits, r0.policy_logits, f"{tag} init policy")
    close(g0.value, r0.value, f"{tag} init value logits")
    close(g0.value_scalar, scalar(r0.value), f"{tag} init value", 2e-4, 2e-4)
    close(g1.latent_state, r1.latent_state, f"{tag} rec latent")
    close(g1.policy_logits, r1.policy_logits, f"{tag} rec policy")
    close(g1.value, r1.value, f"{tag} rec value logits")
    close(g1.value_prefix, r1.value_prefix, f"{tag} rec value prefix logits")
    close(g1.reward_hidden_state[0], r1.reward_hidden_state[0], f"{tag} h'")
    close(g1.reward_hidden_state[1], r1.reward_hidden_state[1], f"{tag} c'")
    close(g1.value_scalar, scalar(r1.value), f"{tag} rec value", 2e-4, 2e-4)
    close(g1.value_prefix_scalar, scalar(r1.value_prefix), f"{tag} value prefix", 2e-4, 2e-4)


@pytest.mark.parametrize("name", NAMES)
def test_model_against_fixture(name):
    import os
    d = np.load(os.path.join(ROOT, "tests", "golden", f"mlp_ez_{name}.npz"))
    _, cu = make(name, int(d["seed"]))
    obs, action = torch.from_numpy(d["obs"]).cuda(), torch.from_numpy(d["action"]).cuda()
    h0, c0 = torch.from_numpy(d["h0"]).cuda(), torch.from_numpy(d["c0"]).cuda()
    g0 = cu.initial_inference(obs, return_scalar_value=True)
    g1 = cu.recurrent_inference(torch.from_numpy(d["init_latent_state"]).cuda(), (h0, c0), action, return_scalars=True)
    close(g0.latent_state, d["init_latent_state"], "init latent")
    close(g0.policy_logits, d["init_policy_logits"], "init policy")
    close(g0.value, d["init_value"], "init value logits")
    close(g0.value_scalar, scalar(d["init_value"]), "init value", 2e-4, 2e-4)
    close(g1.latent_state, d["rec_latent_state"], "rec latent")
    close(g1.policy_logits, d["rec_policy_logits"], "rec policy")
    close(g1.value, d["rec_value"], "rec value logits")
    close(g1.value_prefix, d["rec_value_prefix"], "rec value prefix")
    close(g1.reward_hidden_state[0], d["rec_h"], "h'")
    close(g1.reward_hidden_state[1], d["rec_c"], "c'")
    close(g1.value_prefix_scalar, scalar(d["rec_value_prefix"]), "value prefix", 2e-4, 2e-4)


@pytest.mark.parametrize("name", NAMES)
def test_model_against_restatement_at_every_batch(name):
    from lightzero_b200 import cabi
    ref, cu = make(name, 3)
    partial = []
    for B in BATCHES:
        obs, action, h0, c0 = inputs(name, B, 100 + B)
        check(*run_both(ref, cu, obs, action, h0, c0), f"{name} B={B}")
        L, K, A = cu.latent_state_dim, cu.value_support_size, cu.action_space_size
        for which, x in ((1, obs.cuda()), (0, torch.zeros(B, L, device="cuda"))):
            D = 4 if which or not MR.CONFIGS[name][4] else 6
            info = (cabi.ctypes.c_int32 * 8)()
            out = torch.empty(B * (K + A + 1 + 2 * L), device="cuda")
            cabi.check(cu._lib.lz_model_debug_net_stage(cu._h, which, B, x.data_ptr(), action.cuda().to(torch.int32).data_ptr(), D,
                                                        out.data_ptr(), out.numel() * 4, info, cabi.stream_ptr()), "debug_net_stage")
            p = list(info)
            print(f"[mlp-ez plan] {name} which={which} B={B}: R={p[0]} ctas={p[1]} last={p[2]} layers={p[3]} smem={p[5]} stages={p[6]}")
            assert p[1] == -(-B // p[0]) and p[2] == B - (p[1] - 1) * p[0] and p[7] == D
            partial.append(p[2] < p[0])
    assert any(partial)


@pytest.mark.parametrize("name", ["cartpole", "lunarlander"])
def test_one_root_is_the_same_bits_at_every_slot(name):
    _, cu = make(name, 5)
    obs_dim, A, L, H, _ = MR.CONFIGS[name]
    obs, action, h0, c0 = inputs(name, 200, 9)
    lat = cu.initial_inference(obs.cuda()).latent_state
    t_obs, t_lat, t_act, t_h, t_c = obs[7:8].cuda(), lat[7:8], action[7:8].cuda(), h0[:, 7:8].cuda(), c0[:, 7:8].cuda()

    def run(o, l, a, h, c):
        g0 = cu.initial_inference(o, return_scalar_value=True)
        g1 = cu.recurrent_inference(l, (h, c), a, return_scalars=True)
        return dict(lat0=g0.latent_state, pol0=g0.policy_logits, v0=g0.value_scalar, lat1=g1.latent_state,
                    pol1=g1.policy_logits, vl1=g1.value, vp1=g1.value_prefix, v1=g1.value_scalar, vps=g1.value_prefix_scalar,
                    h=g1.reward_hidden_state[0][0], c=g1.reward_hidden_state[1][0])
    alone = run(t_obs, t_lat, t_act, t_h, t_c)
    for B in (64, 129, 1201):
        pos = sorted({0, 1, 63, 64 % B, B - 1, B // 2, 127 % B})
        o, l = obs[:1].repeat(B, 1).cuda() * 0.5, lat[:1].repeat(B, 1) * 0.5
        a = (torch.arange(B) % A).cuda()
        h, c = torch.zeros(1, B, H, device="cuda"), torch.ones(1, B, H, device="cuda")
        o[pos], l[pos], a[pos], h[:, pos], c[:, pos] = t_obs, t_lat, t_act, t_h, t_c
        got = run(o, l, a, h, c)
        for k, v in got.items():
            same = (v[pos].reshape(len(pos), -1).view(torch.int32) == alone[k].reshape(1, -1).view(torch.int32)).all(1)
            assert same.all(), (B, k, [p for p, s in zip(pos, same.tolist()) if not s])


# ------------------------------------------------------------------------------------------------ searches
def _mcts(S, det, horizon, **kw):
    import lightzero_b200 as lzb
    return lzb.EfficientZeroMCTSCtree(dict(dict(num_simulations=S, deterministic=det, discount_factor=0.997,
                                                lstm_horizon_len=horizon), **kw))


def _search_case(name, B, S, horizon, det, discount=0.997, ikw=None, mutate=None, seed=0):
    """the fused search and the oracle drive on one model; `mutate(ref)` edits the weights before they are loaded"""
    ref, cu = make(name, seed)
    if mutate is not None:
        mutate(ref)
        cu.load_state_dict(ref.state_dict())
    A, H = cu.action_space_size, cu.lstm_hidden_size
    obs, _, h0, c0 = inputs(name, B, seed + 11)
    lat = cu.initial_inference(obs.cuda()).latent_state
    h0, c0 = h0[0].cuda(), c0[0].cuda()
    legal, logits, noises, tp = _inputs(B, A, seed + 5, "1p", **(ikw or {}))
    mcts = _mcts(S, det, horizon, discount_factor=discount)
    roots = mcts.roots(B, legal)
    _prepare(roots, logits, noises, tp)
    mcts.search(roots, cu, lat, (h0[None], c0[None]), tp)
    got, key = readout(roots, A, S), debug_rng(roots)
    nk = mcts.last_num_kernels
    roots.clear()
    from oracle import ctree_port_ez as port
    c = dict(B=B, A=A, S=S, legal=legal, root_logits=logits, noises=noises, to_play=tp, discount=discount, delta=0.01,
             lstm_horizon_len=horizon)
    setup = None if det else (lambda r: r.set_tie_hash(key[0], key[1], 0))
    exp, roots2 = drive(port, c, "ez", network(cu, lat, (h0, c0)), setup=setup)
    return got, exp, nk, roots2.tie_stats(), int(exp["is_reset"].sum()), legal


SEARCHES = {
    # name: config, B, S, horizon, deterministic, discount, input kwargs, policy mutation
    "cartpole_b8_s25_h5_det": ("cartpole", 8, 25, 5, True, 0.997, None, None),
    "cartpole_b65_s25_h1_sto": ("cartpole", 65, 25, 1, False, 0.997, None, None),
    "lunarlander_b130_s50_h3_sto": ("lunarlander", 130, 50, 3, False, 0.997, None, None),
    "lunarlander_b64_s30_h5_sto_tied_d1": ("lunarlander", 64, 30, 5, False, 1.0, dict(noise=False, tie_root=True), zero_policy),
    "bipedalwalker_a256_b40_s20_h5_det": ("bipedalwalker", 40, 20, 5, True, 0.997, None, None),
    "l96_h48_b100_s30_h3_sto": ("l96_h48", 100, 30, 3, False, 1.0, None, None),
}


@pytest.mark.parametrize("case", list(SEARCHES))
def test_fused_search_equals_oracle_driving_the_same_network(case):
    name, B, S, horizon, det, discount, ikw, mutate = SEARCHES[case]
    seed = sum(map(ord, case)) % 97
    got, exp, nk, st, resets, legal = _search_case(name, B, S, horizon, det, discount, ikw, mutate, seed)
    print(f"\n[mlp-ez-search] {case}: resets={resets} ties={st['ties']} draws={st['draws']} kernels={nk}")
    assert_same(got, exp)
    assert visits_sum_to(got, S)
    assert nk == 1 + 4 * S
    assert min(len(l) for l in legal) == 1 or (ikw or {}).get("masks") is False or (ikw or {}).get("tie_root")
    if not det:
        assert st["ties"] > 0 and st["draws"] > 0
    if horizon == 1:
        assert resets == B * S
    elif S > 1:
        assert resets > 0


def test_search_with_reuse_equals_stepwise_drive():
    """ReZero on the value-prefix trees (lunarlander_disc_rezero_ez's model) against ez_tree driven step by step"""
    from lightzero_b200 import ez_tree
    B, S, H = 24, 30, 5
    _, cu = make("lunarlander", 4)
    A = cu.action_space_size
    obs, _, h0, c0 = inputs("lunarlander", B, 4)
    out = cu.initial_inference(obs.cuda())
    h0, c0 = h0[0].cuda(), c0[0].cuda()
    legal, _, noises, tp = _inputs(B, A, 9, "1p")
    rng = np.random.default_rng(3)
    true_action = [int(l[rng.integers(len(l))]) for l in legal]
    reuse_value = (rng.standard_normal(B) * 0.5).astype(np.float32).tolist()
    mcts = _mcts(S, True, H)
    roots = mcts.roots(B, legal)
    roots.prepare(0.25, noises, [0.] * B, out.policy_logits, tp)
    mcts.search_with_reuse(roots, cu, out.latent_state, (h0[None], c0[None]), tp, true_action, reuse_value)
    fused = readout(roots, A, S)
    roots.clear()
    c = dict(B=B, A=A, S=S, legal=legal, root_logits=out.policy_logits.cpu().numpy(), noises=noises, to_play=tp,
             true_action=true_action, reuse_value=reuse_value, lstm_horizon_len=H)
    step, _ = drive(ez_tree, c, "ez_reuse", network(cu, out.latent_state, (h0, c0)))
    assert_same(step, fused)
    assert min(step["n_inferred"].tolist()) < B


def test_collect_equals_initial_inference_prepare_and_search():
    import lightzero_b200 as lzb
    from lightzero_b200.collect import EfficientZeroCollectPolicy
    name, B, S = "cartpole", 16, 25
    _, cu = make(name, 8)
    A = cu.action_space_size
    obs, _, _, _ = inputs(name, B, 8)
    legal, _, noises, tp = _inputs(B, A, 13, "1p", masks=False)
    mask = np.ones((B, A), np.uint8)
    noise_rows = np.asarray(noises, np.float32)
    cfg = dict(num_simulations=S, discount_factor=0.997, lstm_horizon_len=5)
    pol = EfficientZeroCollectPolicy(cu, cfg)
    got = pol.search_batch(obs.cuda(), mask, noise_rows, tp, read_back=False)
    out = cu.initial_inference(obs.cuda(), return_scalar_value=True)
    mcts = lzb.EfficientZeroMCTSCtree(cfg)
    roots = mcts.roots(B, legal)
    roots.prepare(0.25, noises, [0.] * B, out.policy_logits, tp)
    mcts.search(roots, cu, out.latent_state, out.reward_hidden_state, tp)
    exp = readout(roots, A, S)
    roots.clear()
    assert torch.equal(got["pred_value"].cpu(), out.value_scalar.cpu())
    assert torch.equal(got["policy_logits"].cpu(), out.policy_logits.cpu())
    assert np.array_equal(got["visits"].cpu().numpy(), exp["distributions"])
    assert np.array_equal(got["values"].cpu().numpy().view(np.uint32), exp["root_values_bits"])
    host = pol.search_batch(obs, mask, noise_rows, tp)             # host observations: the chunked copy path
    assert np.array_equal(host["visits"].numpy(), exp["distributions"])


def test_reanalyze_runs_with_the_model():
    import lightzero_b200 as lzb
    from lightzero_b200.reanalyze import compute_target_policy_reanalyzed
    name, segments, unroll = "lunarlander", 6, 5
    _, cu = make(name, 2)
    A = cu.action_space_size
    T = segments * (unroll + 1)
    obs, _, _, _ = inputs(name, T, 2)
    mask = np.ones((T, A), np.uint8)
    mcts = lzb.EfficientZeroMCTSCtree(dict(num_simulations=16, lstm_horizon_len=5))
    out = compute_target_policy_reanalyzed(cu, mcts, obs.cuda(), mask, [-1] * T, [1] * T, list(range(segments)),
                                           num_unroll_steps=unroll, action_space_size=A, reanalyze_noise=False)
    assert out.shape == (segments, unroll + 1, A)
    assert np.allclose(out.sum(-1), 1.0)


def test_refusals():
    import lightzero_b200 as lzb
    from lightzero_b200 import cabi
    bad = [dict(latent_state_dim=48), dict(latent_state_dim=288), dict(lstm_hidden_size=40), dict(lstm_hidden_size=528),
           dict(observation_shape=4097), dict(action_space_size=609), dict(value_head_hidden_channels=[33]),
           dict(reward_support_range=(-400., 401., 1.), value_support_range=(-400., 401., 1.))]
    msgs = ["latent_dim", "latent_dim", "lstm_hidden_size", "lstm_hidden_size", "obs_dim", "action_space_size", "hidden",
            "support size"]
    for kw, msg in zip(bad, msgs):
        with pytest.raises(cabi.LzError, match=msg):
            lzb.EfficientZeroModelMLP(**dict(dict(observation_shape=4, action_space_size=2, latent_state_dim=128,
                                                  lstm_hidden_size=128), **kw))
    for kw in (dict(discrete_action_encoding_type="not_one_hot"), dict(norm_type="LN"), dict(state_norm=True)):
        with pytest.raises(NotImplementedError):
            lzb.EfficientZeroModelMLP(observation_shape=4, action_space_size=2, latent_state_dim=128, lstm_hidden_size=128, **kw)
    _, cu = make("cartpole", 1)
    mz = lzb.MuZeroMCTSCtree(dict(num_simulations=4))
    r = mz.roots(1, [[0, 1]])
    r.prepare_no_noise([0.], np.zeros((1, 2), np.float32), [-1])
    with pytest.raises(TypeError, match="EfficientZeroMCTSCtree"):
        mz.search(r, cu, torch.zeros(1, 128, device="cuda"), [-1])
    r.clear()
    with pytest.raises(TypeError, match="Gumbel"):
        g = lzb.GumbelMuZeroMCTSCtree(dict(num_simulations=4))
        g.search(g.roots(1, [[0, 1]]), cu, torch.zeros(1, 128, device="cuda"), [-1])
    # uint8 frames are the Atari path: the MLP model refuses them
    mcts = _mcts(4, True, 5)
    roots = mcts.roots(2, [[0, 1]] * 2)
    roots.prepare_no_noise([0.] * 2, np.zeros((2, 2), np.float32), [-1, -1])
    roots._ez, roots._lstm_horizon = True, 5
    roots._materialize(4)
    t = roots._tree
    q = t.search_for(cu, 4, (1, 5))
    frames = torch.zeros(2, 4, dtype=torch.uint8, device="cuda")
    rc = cu._lib.lz_search_collect_u8(q, frames.data_ptr(), None, None, 0.0, None, 1, None, None, cabi.stream_ptr())
    assert rc == -1 and b"conv model" in cu._lib.lz_last_error()
    roots.clear()
