"""GPU tests of MuZeroModelMLP on the tensor-core MLP kernel (csrc/mlp_tc.cu, model kind 4: the configs the fp32 kernels of
csrc/mlp.cu do not take, lunarlander MuZero and ReZero-MuZero with latent 256 among them):
- the CUDA model against the reference class's fixtures and the PyTorch restatement at B in {1, 63, 64, 65, 1024}: tc3 within
  1e-5 on latents and logits, 2e-4 on the scalars; tc1 within its stated looser bound;
- one root gives the same bits at every row of a CTA;
- the fused multi-kernel search, search_with_reuse, the Gumbel search, collect and reanalyze against the oracle driving the
  same network (or the manual restatement), bit for bit;
- the reference's lunarlander MuZero model config, passed as keywords, constructs and searches;
- the refusals of the accepted space, and the configs the fp32 kernels take stay there."""
import os

import numpy as np
import pytest
import torch

import mlp_mz_model_ref as MR
from conftest import ROOT
from oracle.tree_drive import assert_same, drive, network, readout
from test_gpu_search_oracle import _inputs, fused_search, oracle_search, visits_sum_to

pytestmark = pytest.mark.gpu

NAMES = list(MR.CONFIGS)
BATCHES = (1, 63, 64, 65, 1024)
TC1_TOL = 2e-2          # tc1 (one fp16 pass): not the parity mode; latents and logits within 2e-2, scalars within 0.1


def make(name, seed=0, math="tc3", ssl_keys=True):
    """(restatement on the CPU, CUDA model loaded from its state_dict); SSL head keys ride along and are ignored"""
    import lightzero_b200 as lzb
    ref = MR.build(name, seed)
    sd = dict(ref.state_dict())
    if ssl_keys:
        sd["projection.0.weight"] = torch.randn(8, 8)
    cu = lzb.MuZeroModelMLP(**MR.model_kwargs(name)).load_state_dict(sd)
    cu.set_math(math)
    return ref, cu


def close(got, exp, what, atol=1e-5, rtol=1e-5):
    got, exp = torch.as_tensor(got).double().cpu(), torch.as_tensor(exp).double().cpu()
    err = ((got - exp).abs() - rtol * exp.abs()).max().item()
    assert err <= atol, f"{what}: max excess error {err:.3g}"
    return err


def inputs(name, B, seed):
    obs_dim, A = MR.CONFIGS[name][:2]
    g = torch.Generator().manual_seed(seed)
    obs = torch.rand((B, obs_dim), generator=g) * 2.0 - 1.0
    action = torch.randint(0, A, (B,), generator=g)
    return obs, action


def run_both(ref, cu, obs, action):
    with torch.no_grad():
        r0 = ref.initial_inference(obs)
        r1 = ref.recurrent_inference(r0.latent_state, action)
    g0 = cu.initial_inference(obs.cuda(), return_scalar_value=True)
    g1 = cu.recurrent_inference(r0.latent_state.cuda(), action.cuda(), return_scalars=True)
    return r0, r1, g0, g1


def check(name, r0, r1, g0, g1, tag, tol=1e-5, stol=2e-4):
    sup = MR.CONFIGS[name][5]
    close(g0.latent_state, r0.latent_state, f"{tag} init latent", tol, tol)
    close(g0.policy_logits, r0.policy_logits, f"{tag} init policy", tol, tol)
    close(g0.value, r0.value, f"{tag} init value logits", tol, tol)
    close(g0.value_scalar, MR.scalar(r0.value, sup), f"{tag} init value", stol, stol)
    close(g1.latent_state, r1.latent_state, f"{tag} rec latent", tol, tol)
    close(g1.policy_logits, r1.policy_logits, f"{tag} rec policy", tol, tol)
    close(g1.value, r1.value, f"{tag} rec value logits", tol, tol)
    close(g1.reward, r1.reward, f"{tag} rec reward logits", tol, tol)
    close(g1.value_scalar, MR.scalar(r1.value, sup), f"{tag} rec value", stol, stol)
    close(g1.reward_scalar, MR.scalar(r1.reward, sup), f"{tag} rec reward", stol, stol)


@pytest.mark.parametrize("name", NAMES)
def test_model_against_fixture(name):
    d = np.load(os.path.join(ROOT, "tests", "golden", f"mlp_mz_{name}.npz"))
    _, cu = make(name, int(d["seed"]))
    sup = MR.CONFIGS[name][5]
    obs, action = torch.from_numpy(d["obs"]).cuda(), torch.from_numpy(d["action"]).cuda()
    g0 = cu.initial_inference(obs, return_scalar_value=True)
    g1 = cu.recurrent_inference(torch.from_numpy(d["init_latent_state"]).cuda(), action, return_scalars=True)
    close(g0.latent_state, d["init_latent_state"], "init latent")
    close(g0.policy_logits, d["init_policy_logits"], "init policy")
    close(g0.value, d["init_value"], "init value logits")
    close(g0.value_scalar, MR.scalar(d["init_value"], sup), "init value", 2e-4, 2e-4)
    close(g1.latent_state, d["rec_latent_state"], "rec latent")
    close(g1.policy_logits, d["rec_policy_logits"], "rec policy")
    close(g1.value, d["rec_value"], "rec value logits")
    close(g1.reward, d["rec_reward"], "rec reward logits")
    close(g1.reward_scalar, MR.scalar(d["rec_reward"], sup), "rec reward", 2e-4, 2e-4)
    close(g1.value_scalar, MR.scalar(d["rec_value"], sup), "rec value", 2e-4, 2e-4)


@pytest.mark.parametrize("name", NAMES)
def test_model_against_restatement_at_every_batch(name):
    from lightzero_b200 import cabi
    ref, cu = make(name, 3)
    L, K, A = cu.latent_state_dim, cu.value_support_size, cu.action_space_size
    res = MR.CONFIGS[name][3]
    for B in BATCHES:
        obs, action = inputs(name, B, 100 + B)
        check(name, *run_both(ref, cu, obs, action), f"{name} B={B}")
        for which, x in ((1, obs.cuda()), (0, torch.zeros(B, L, device="cuda"))):
            D = 4 if which else (6 if res else 4)       # dense layers: dynamics (4 or 2) + prediction common (2)
            info = (cabi.ctypes.c_int32 * 8)()
            out = torch.empty(B * (2 * K + A + 2 + 2 * L), device="cuda")
            cabi.check(cu._lib.lz_model_debug_net_stage(cu._h, which, B, x.data_ptr(), action.cuda().to(torch.int32).data_ptr(), D,
                                                        out.data_ptr(), out.numel() * 4, info, cabi.stream_ptr()), "debug_net_stage")
            p = list(info)
            print(f"[mlp-mz plan] {name} which={which} B={B}: R={p[0]} ctas={p[1]} last={p[2]} layers={p[3]} smem={p[5]} stages={p[6]}")
            assert p[1] == -(-B // p[0]) and p[2] == B - (p[1] - 1) * p[0] and p[7] == D and p[4] == 3


@pytest.mark.parametrize("name", NAMES)
def test_tc1_within_its_looser_bound(name):
    ref, cu = make(name, 3, math="tc1")
    obs, action = inputs(name, 65, 7)
    check(name, *run_both(ref, cu, obs, action), f"{name} tc1", TC1_TOL, 0.1)


@pytest.mark.parametrize("name", ["lunarlander", "l160_a18"])
def test_one_root_is_the_same_bits_at_every_row(name):
    _, cu = make(name, 5)
    A = MR.CONFIGS[name][1]
    obs, action = inputs(name, 200, 9)
    lat = cu.initial_inference(obs.cuda()).latent_state
    t_obs, t_lat, t_act = obs[7:8].cuda(), lat[7:8], action[7:8].cuda()

    def run(o, l, a):
        g0 = cu.initial_inference(o, return_scalar_value=True)
        g1 = cu.recurrent_inference(l, a, return_scalars=True)
        return dict(lat0=g0.latent_state, pol0=g0.policy_logits, v0=g0.value_scalar, lat1=g1.latent_state,
                    pol1=g1.policy_logits, vl1=g1.value, rl1=g1.reward, v1=g1.value_scalar, r1=g1.reward_scalar)
    alone = run(t_obs, t_lat, t_act)
    for B in (64, 129, 1201):
        pos = sorted({0, 1, 63, 64 % B, B - 1, B // 2, 127 % B})
        o, l = obs[:1].repeat(B, 1).cuda() * 0.5, lat[:1].repeat(B, 1) * 0.5
        a = (torch.arange(B) % A).cuda()
        o[pos], l[pos], a[pos] = t_obs, t_lat, t_act
        got = run(o, l, a)
        for k, v in got.items():
            same = (v[pos].reshape(len(pos), -1).view(torch.int32) == alone[k].reshape(1, -1).view(torch.int32)).all(1)
            assert same.all(), (B, k, [p for p, s in zip(pos, same.tolist()) if not s])


# ------------------------------------------------------------------------------------------------ searches
@torch.no_grad()
def zero_policy(ref):
    """policy FC2 weights and bias zero: every prior is uniform, unvisited siblings tie exactly"""
    fc = ref.prediction_network.fc_policy_head[-1]
    fc.weight.zero_()
    fc.bias.zero_()


SEARCHES = {
    # name: config, B, S, deterministic, players, input kwargs, policy mutation
    "lunarlander_b8_s50_det": ("lunarlander", 8, 50, True, "1p", {}, None),
    "lunarlander_b256_s50_det": ("lunarlander", 256, 50, True, "1p", {}, None),
    "lunarlander_b8_s50_sto": ("lunarlander", 8, 50, False, "1p", {}, None),
    "lunarlander_b256_s50_sto_tied": ("lunarlander", 256, 50, False, "1p", dict(noise=False, tie_root=True), zero_policy),
    "l160_a18_b65_s30_sto_2p": ("l160_a18", 65, 30, False, "2p", {}, None),
    "l224_wide_b40_s20_det_tc1": ("l224_wide", 40, 20, True, "mixed", {}, None),
}


@pytest.mark.parametrize("case", list(SEARCHES))
def test_fused_search_equals_oracle_driving_the_same_network(case):
    import lightzero_b200 as lzb
    name, B, S, det, players, ikw, mutate = SEARCHES[case]
    seed = sum(map(ord, case)) % 97
    ref, cu = make(name, seed, math="tc1" if case.endswith("tc1") else "tc3")
    if mutate is not None:
        mutate(ref)
        cu.load_state_dict(ref.state_dict())
    A = cu.action_space_size
    obs, _ = inputs(name, B, seed + 11)
    latent = cu.initial_inference(obs.cuda()).latent_state
    legal, logits, noises, tp = _inputs(B, A, seed + 5, players, **ikw)
    mcts = lzb.MuZeroMCTSCtree(dict(num_simulations=S, deterministic=det, discount_factor=0.997))
    got, key, plan, roots = fused_search(cu, mcts, S, latent, legal, logits, noises, tp)
    exp, st = oracle_search(cu, S, latent, legal, logits, noises, tp, det, key=key)
    kernels = mcts.last_num_kernels
    roots.clear()
    print(f"\n[mlp-mz-search] {case}: ties={st['ties']} draws={st['draws']} kernels={kernels}")
    assert_same(got, exp)
    assert visits_sum_to(got, S)
    assert not plan["persistent"] and kernels == 2 * S + 1
    if not det:
        assert st["ties"] > 0 and st["draws"] > 0


def test_search_with_reuse_equals_stepwise_drive():
    """ReZero-MuZero (lunarlander_disc_rezero_mz_config.py's model) against mz_tree driven step by step"""
    import lightzero_b200 as lzb
    from lightzero_b200 import mz_tree
    B, S = 24, 30
    _, cu = make("lunarlander", 4)
    A = cu.action_space_size
    obs, _ = inputs("lunarlander", B, 4)
    out = cu.initial_inference(obs.cuda())
    legal, _, noises, tp = _inputs(B, A, 9, "1p")
    rng = np.random.default_rng(3)
    true_action = [int(l[rng.integers(len(l))]) for l in legal]
    reuse_value = (rng.standard_normal(B) * 0.5).astype(np.float32).tolist()
    mcts = lzb.MuZeroMCTSCtree(dict(num_simulations=S, deterministic=True, discount_factor=0.997))
    roots = mcts.roots(B, legal)
    roots.prepare(0.25, noises, [0.] * B, out.policy_logits, tp)
    mcts.search_with_reuse(roots, cu, out.latent_state, tp, true_action, reuse_value)
    fused = readout(roots, A, S)
    kernels = mcts.last_num_kernels
    roots.clear()
    c = dict(B=B, A=A, S=S, legal=legal, root_logits=out.policy_logits.cpu().numpy(), noises=noises, to_play=tp,
             true_action=true_action, reuse_value=reuse_value)
    step, _ = drive(mz_tree, c, "reuse", network(cu, out.latent_state))
    assert_same(step, fused)
    assert min(step["n_inferred"].tolist()) < B
    assert kernels >= 1 + S


@pytest.mark.parametrize("name,B,m", [("lunarlander", 64, 4), ("l160_a18", 131, 8)])
def test_gumbel_search_equals_reference_tree(name, B, m):
    import lightzero_b200 as lzb
    from oracle import build_gmz_ref
    gref = build_gmz_ref.load()
    if gref is None:
        pytest.skip("compiled reference Gumbel tree not built (oracle/build_gmz_ref.py)")
    S = 32
    _, cu = make(name, 6)
    A = cu.action_space_size
    obs, _ = inputs(name, B, 6)
    out = cu.initial_inference(obs.cuda(), return_scalar_value=True)
    legal, _, noises, tp = _inputs(B, A, 12, "1p")
    gmcts = lzb.GumbelMuZeroMCTSCtree(dict(num_simulations=S, max_num_considered_actions=m))
    roots = gmcts.roots(B, legal)
    roots.prepare(0.25, noises, [0.] * B, out.value_scalar, out.policy_logits, tp)
    gmcts.search(roots, cu, out.latent_state, tp)
    got = readout(roots, A, S, 0.997)
    kernels = gmcts.last_num_kernels
    roots.clear()
    c = dict(B=B, A=A, S=S, legal=legal, root_logits=out.policy_logits.cpu().numpy(), noises=noises, to_play=tp, m=m,
             root_values=out.value_scalar.cpu().numpy())
    exp, _ = drive(gref, c, "gumbel", network(cu, out.latent_state))
    assert_same(got, exp)
    assert kernels >= 1 + 2 * S


def test_collect_equals_initial_inference_prepare_and_search():
    import lightzero_b200 as lzb
    from lightzero_b200.collect import MuZeroCollectPolicy
    name, B, S = "lunarlander", 16, 25
    _, cu = make(name, 8)
    A = cu.action_space_size
    obs, _ = inputs(name, B, 8)
    legal, _, noises, tp = _inputs(B, A, 13, "1p")
    mask = np.zeros((B, A), np.uint8)
    for b, l in enumerate(legal):
        mask[b, l] = 1
    noise_rows = np.zeros((B, A), np.float32)
    for b, n in enumerate(noises):
        noise_rows[b, :len(n)] = n
    cfg = dict(num_simulations=S, deterministic=True, discount_factor=0.997)
    pol = MuZeroCollectPolicy(cu, cfg)
    got = pol.search_batch(obs.cuda(), mask, noise_rows, tp, read_back=False)
    out = cu.initial_inference(obs.cuda(), return_scalar_value=True)
    mcts = lzb.MuZeroMCTSCtree(cfg)
    roots = mcts.roots(B, legal)
    roots.prepare(0.25, noises, [0.] * B, out.policy_logits, tp)
    mcts.search(roots, cu, out.latent_state, tp)
    exp = readout(roots, A, S)
    roots.clear()
    assert torch.equal(got["pred_value"].cpu(), out.value_scalar.cpu())
    assert torch.equal(got["policy_logits"].cpu(), out.policy_logits.cpu())
    assert np.array_equal(got["visits"].cpu().numpy(), exp["distributions"])
    assert np.array_equal(got["values"].cpu().numpy().view(np.uint32), exp["root_values_bits"])
    host = pol.search_batch(obs, mask, noise_rows, tp)             # host observations: lz_search_collect_host's chunked copies
    assert np.array_equal(host["visits"].numpy(), exp["distributions"])


def test_reanalyze_equals_its_manual_restatement():
    """one compute_target_policy_reanalyzed call against initial_inference + prepare + search + the target assembly"""
    import lightzero_b200 as lzb
    from lightzero_b200.reanalyze import compute_target_policy_reanalyzed
    name, segments, unroll, S = "lunarlander", 6, 5, 16
    _, cu = make(name, 2)
    A = cu.action_space_size
    T = segments * (unroll + 1)
    obs, _ = inputs(name, T, 2)
    mask = np.ones((T, A), np.uint8)
    rng = np.random.default_rng(2)
    noises = np.stack([rng.dirichlet([0.3] * A).astype(np.float32) for _ in range(T)])
    policy_mask = [1] * (T - 2) + [0] * 2
    cfg = dict(num_simulations=S, deterministic=True, discount_factor=0.997)
    got, got_values, roots = compute_target_policy_reanalyzed(
        cu, lzb.MuZeroMCTSCtree(cfg), obs.cuda(), mask, [-1] * T, policy_mask, list(range(segments)), num_unroll_steps=unroll,
        action_space_size=A, noises=noises, return_roots=True)
    roots.clear()
    out = cu.initial_inference(obs.cuda())
    mcts = lzb.MuZeroMCTSCtree(cfg)
    roots = mcts.roots(T, [list(range(A))] * T)
    roots.prepare(0.25, noises, [0.] * T, out.policy_logits, [-1] * T)
    mcts.search(roots, cu, out.latent_state, [-1] * T)
    dist, values = np.asarray(roots.get_distributions(), np.float64), roots.get_values()
    roots.clear()
    exp = np.where(np.asarray(policy_mask)[:, None] == 1, dist / dist.sum(1, keepdims=True), 0.0).reshape(segments, unroll + 1, A)
    assert got.shape == (segments, unroll + 1, A)
    assert np.array_equal(got, exp)
    assert np.array_equal(np.asarray(got_values, np.float32).view(np.uint32), np.asarray(values, np.float32).view(np.uint32))


def test_reference_lunarlander_config_constructs_and_searches():
    """the model= dict of zoo/box2d/lunarlander/config/lunarlander_disc_muzero_config.py, passed as keywords, and a
    state_dict with the SSL heads it builds (self_supervised_learning_loss=True): ignored at inference"""
    import lightzero_b200 as lzb
    model_cfg = dict(observation_shape=8, action_space_size=4, model_type='mlp', lstm_hidden_size=256, latent_state_dim=256,
                     self_supervised_learning_loss=True, discrete_action_encoding_type='one_hot',
                     res_connection_in_dynamics=True, norm_type='BN')
    ref = MR.build("lunarlander", 1)
    sd = dict(ref.state_dict())
    sd.update({"projection.0.weight": torch.randn(1024, 256), "prediction_head.0.weight": torch.randn(512, 1024)})
    cu = lzb.MuZeroModelMLP(**model_cfg).load_state_dict(sd)
    B, S = 8, 50
    obs, _ = inputs("lunarlander", B, 1)
    out = cu.initial_inference(obs.cuda())
    with torch.no_grad():
        exp = ref.initial_inference(obs)
    close(out.latent_state, exp.latent_state, "latent")
    mcts = lzb.MuZeroMCTSCtree(dict(num_simulations=S))
    roots = mcts.roots(B, [[0, 1, 2, 3]] * B)
    roots.prepare_no_noise([0.] * B, out.policy_logits, [-1] * B)
    mcts.search(roots, cu, out.latent_state, [-1] * B)
    assert all(sum(d) == S for d in roots.get_distributions())
    roots.clear()


def test_refusals_and_kind_selection():
    import lightzero_b200 as lzb
    from lightzero_b200 import cabi
    base = dict(observation_shape=8, action_space_size=4, latent_state_dim=256)
    for kw, msg in ((dict(latent_state_dim=512), r"\[32,256\]"), (dict(latent_state_dim=200), "multiple of 32"),
                    (dict(action_space_size=609), r"action_space_size in \[1,608\]")):
        with pytest.raises(cabi.LzError, match=msg) as e:
            lzb.MuZeroModelMLP(**dict(base, **kw))
        assert "fp32 MLP kernels" in str(e.value) and "tensor-core MLP kernel" in str(e.value)
    with pytest.raises(cabi.LzError, match="support size"):
        lzb.MuZeroModelMLP(**dict(base, reward_support_range=(-400., 401., 1.), value_support_range=(-400., 401., 1.)))
    for kw in (dict(discrete_action_encoding_type="not_one_hot"), dict(norm_type="LN"), dict(state_norm=True),
               dict(categorical_distribution=False)):
        with pytest.raises(NotImplementedError):
            lzb.MuZeroModelMLP(**base, **kw)
    # a config the fp32 kernels take stays on them: no math mode
    cart = lzb.MuZeroModelMLP(observation_shape=4, action_space_size=2, latent_state_dim=128)
    with pytest.raises(cabi.LzError, match="no math mode"):
        cart.set_math("tc1")
    with pytest.raises(ValueError, match="tc3"):
        cart.set_math("fp64")
    # and one they do not take runs on the tensor cores: tc1 / tc3 switch
    wide = lzb.MuZeroModelMLP(observation_shape=200, action_space_size=2, latent_state_dim=128)
    wide.set_math("tc1").set_math("tc3")
