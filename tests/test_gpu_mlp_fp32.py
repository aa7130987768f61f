"""GPU tests of MuZeroModelMLP on the fp32 MLP kernels (csrc/mlp.cu, model kind 1: latents up to 128, the reference's
vector-observation MuZero configs), at every config of tests/mlp_fp32_model_ref.py:
- the CUDA model against the reference class's fixtures and the PyTorch restatement at B = 1 .. 1201 (every B mod 4, the
  kernels' roots per CTA): within 1e-5 on latents and logits, 2e-4 on the scalars;
- one root gives the same bits in every slot of a CTA;
- the fused multi-kernel search, search_with_reuse, the Gumbel search, collect and reanalyze against the oracle driving the
  same network (or the manual restatement), bit for bit;
- the reference's model dicts, passed as keywords with their SSL keys, construct and search;
- every config stays on the fp32 kernels, one step past each edge of their envelope does not, and a head with two hidden
  layers is refused at finalize."""
import os

import numpy as np
import pytest
import torch

import mlp_fp32_model_ref as MR
from conftest import ROOT
from oracle.tree_drive import assert_same, drive, network, readout
from test_gpu_mlp_mz import close, run_both, zero_policy
from test_gpu_search_oracle import _inputs, fused_search, oracle_search, visits_sum_to

pytestmark = pytest.mark.gpu

NAMES = list(MR.CONFIGS)
BATCHES = (1, 2, 3, 4, 5, 131, 1023, 1024, 1201)


def make(name, seed=0, ssl_keys=True):
    """(restatement on the CPU, CUDA model loaded from its state_dict); SSL head keys ride along and are ignored"""
    import lightzero_b200 as lzb
    ref = MR.build(name, seed)
    sd = dict(ref.state_dict())
    if ssl_keys:
        sd["projection.0.weight"] = torch.randn(8, 8)
    cu = lzb.MuZeroModelMLP(**MR.model_kwargs(name)).load_state_dict(sd)
    return ref, cu


def inputs(name, B, seed):
    """seeded observations in [-1, 1) and actions; the last action of the space is always among them"""
    obs_dim, A = MR.CONFIGS[name][:2]
    g = torch.Generator().manual_seed(seed)
    obs = torch.rand((B, obs_dim), generator=g) * 2.0 - 1.0
    action = torch.randint(0, A, (B,), generator=g)
    action[B // 2] = A - 1
    return obs, action


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


def debug_stage(cu, which, x, action, s):
    """lz_model_debug_net_stage on kind 1: (output rows [B, width] of stage s, or the whole program's flat outputs, h_info)"""
    from lightzero_b200 import cabi
    L, K, A = cu.latent_state_dim, cu.value_support_size, cu.action_space_size
    n = x.shape[0]
    out = torch.full((n * (L + 2 * K + A + 2),), float("nan"), device="cuda")
    info = (cabi.ctypes.c_int32 * 8)()
    cabi.check(cu._lib.lz_model_debug_net_stage(cu._h, which, n, x.contiguous().data_ptr(), action.data_ptr(), s, out.data_ptr(),
                                                out.numel() * 4, info, cabi.stream_ptr()), "lz_model_debug_net_stage")
    torch.cuda.synchronize()
    p = list(info)
    if s < p[3]:
        return out[:n * p[4]].view(n, p[4]), p
    return out, p


@pytest.mark.parametrize("name", NAMES)
def test_model_against_fixture(name):
    d = np.load(os.path.join(ROOT, "tests", "golden", f"mlp_fp32_{name}.npz"))
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
    ref, cu = make(name, 3)
    res = MR.CONFIGS[name][3]
    for B in BATCHES:
        obs, action = inputs(name, B, 100 + B)
        r0, r1, g0, g1 = run_both(ref, cu, obs, action)
        check(name, r0, r1, g0, g1, f"{name} B={B}")
        for which, x in ((1, obs.cuda()), (0, r0.latent_state.cuda())):
            D = 9 if which else (13 if res else 10)
            a = action.cuda().to(torch.int32)
            out, p = debug_stage(cu, which, x, a, D)
            print(f"[mlp-fp32 plan] {name} which={which} B={B}: R={p[0]} ctas={p[1]} last={p[2]} D={p[3]}")
            assert p[0] == 4 and p[1] == -(-B // 4) and p[2] == B - (p[1] - 1) * 4 and p[3] == D
            # the hook's whole-program layout holds the outputs the inference entry points return, bit for bit
            L, K, A = cu.latent_state_dim, cu.value_support_size, cu.action_space_size
            g = g0 if which else g1
            lat, vl = out[:B * L].view(B, L), out[B * L:B * (L + K)].view(B, K)
            pl, v = out[B * (L + K):B * (L + K + A)].view(B, A), out[B * (L + K + A):B * (L + K + A + 1)]
            assert torch.equal(lat, g.latent_state) and torch.equal(vl, g.value) and torch.equal(pl, g.policy_logits)
            assert torch.equal(v, g.value_scalar)
            if not which:
                rl, r = out[B * (L + K + A + 1):B * (L + 2 * K + A + 1)].view(B, K), out[B * (L + 2 * K + A + 1):B * (L + 2 * K + A + 2)]
                assert torch.equal(rl, g1.reward) and torch.equal(r, g1.reward_scalar)


@pytest.mark.parametrize("name", ["pendulum", "l8_a152", "l100_o160", "l44_half"])
def test_debug_stage_last_layers_are_the_program_outputs(name):
    """the cut after the last layer of each head equals what the production kernels return, at a partial last CTA"""
    _, cu = make(name, 4)
    B = 131
    obs, action = inputs(name, B, 17)
    a = action.cuda().to(torch.int32)
    g0 = cu.initial_inference(obs.cuda())
    g1 = cu.recurrent_inference(g0.latent_state, a)
    res = MR.CONFIGS[name][3]
    for which, x, g, stages in ((1, obs.cuda(), g0, dict(latent=2, value=6, policy=8)),
                                (0, g0.latent_state, g1, dict(latent=2 if res else 1, reward=6 if res else 3,
                                                              value=10 if res else 7, policy=12 if res else 9))):
        for key, s in stages.items():
            got, p = debug_stage(cu, which, x, a, s)
            exp = dict(latent=g.latent_state, value=g.value, policy=g.policy_logits, reward=g.reward if not which else None)[key]
            assert p[2] == 3 and p[4] == exp.shape[1], (which, key, p)
            assert torch.equal(got, exp), (name, which, key)


@pytest.mark.parametrize("name", ["pendulum", "l8_a152", "l100_o160"])
def test_one_root_is_the_same_bits_in_every_slot(name):
    _, cu = make(name, 5)
    A = MR.CONFIGS[name][1]
    obs, action = inputs(name, 200, 9)
    lat = cu.initial_inference(obs.cuda()).latent_state
    t_obs, t_lat, t_act = obs[7:8].cuda(), lat[7:8], action[100:101].cuda()      # action A - 1

    def run(o, l, a):
        g0 = cu.initial_inference(o, return_scalar_value=True)
        g1 = cu.recurrent_inference(l, a, return_scalars=True)
        return dict(lat0=g0.latent_state, pol0=g0.policy_logits, vl0=g0.value, v0=g0.value_scalar, lat1=g1.latent_state,
                    pol1=g1.policy_logits, vl1=g1.value, rl1=g1.reward, v1=g1.value_scalar, r1=g1.reward_scalar)
    alone = run(t_obs, t_lat, t_act)
    for B in (4, 5, 131, 1201):
        pos = sorted({0, 1, 2, 3, B // 2, B - 1, (B - 2) % B})        # every position mod 4 among other roots
        o, l = obs[:1].repeat(B, 1).cuda() * 0.5, lat[:1].repeat(B, 1) * 0.5
        a = (torch.arange(B) % A).cuda()
        o[pos], l[pos], a[pos] = t_obs, t_lat, t_act
        got = run(o, l, a)
        for k, v in got.items():
            same = (v[pos].reshape(len(pos), -1).view(torch.int32) == alone[k].reshape(1, -1).view(torch.int32)).all(1)
            assert same.all(), (B, k, [p for p, s in zip(pos, same.tolist()) if not s])


# ------------------------------------------------------------------------------------------------ searches
SEARCHES = {
    # name: config, B, S, deterministic, players, input kwargs, policy mutation
    "pendulum_b8_s50_det": ("pendulum", 8, 50, True, "1p", {}, None),
    "pendulum_b131_s50_sto_2p": ("pendulum", 131, 50, False, "2p", {}, None),
    "pendulum_b64_s30_sto_tied": ("pendulum", 64, 30, False, "1p", dict(noise=False, tie_root=True), zero_policy),
    "mountain_car_b8_s25_det": ("mountain_car", 8, 25, True, "1p", dict(masks=False), None),
    "mountain_car_b37_s25_sto_mixed": ("mountain_car", 37, 25, False, "mixed", {}, None),
    "l8_a152_b21_s40_sto_2p": ("l8_a152", 21, 40, False, "2p", {}, None),
    "l8_a152_b9_s30_det_tied": ("l8_a152", 9, 30, True, "mixed", dict(noise=False, tie_root=True), zero_policy),
}


@pytest.mark.parametrize("case", list(SEARCHES))
def test_fused_search_equals_oracle_driving_the_same_network(case):
    import lightzero_b200 as lzb
    name, B, S, det, players, ikw, mutate = SEARCHES[case]
    seed = sum(map(ord, case)) % 97
    ref, cu = make(name, seed)
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
    print(f"\n[mlp-fp32-search] {case}: persistent={plan['persistent']} N={plan['N']} kernels={kernels} ties={st['ties']} "
          f"draws={st['draws']} max_len={st['max_len']}")
    assert_same(got, exp)
    assert visits_sum_to(got, S)
    assert not plan["persistent"] and plan["N"] == S + 1 and kernels == 2 * S + 1      # the multi-kernel search graph
    if not det:
        assert st["ties"] > 0 and st["draws"] > 0
    if mutate is not None:
        assert st["ties"] >= B


@pytest.mark.parametrize("name", ["pendulum", "mountain_car"])
def test_search_with_reuse_equals_stepwise_drive(name):
    import lightzero_b200 as lzb
    from lightzero_b200 import mz_tree
    B, S = 24, 30
    _, cu = make(name, 4)
    A = cu.action_space_size
    obs, _ = inputs(name, B, 4)
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


@pytest.mark.parametrize("name,B,m,S", [("pendulum", 64, 11, 50), ("mountain_car", 37, 3, 25)])
def test_gumbel_search_equals_reference_tree(name, B, m, S):
    """pendulum: zoo/classic_control/pendulum/config/pendulum_cont_disc_gumbel_muzero_config.py (S = 50, every action considered)"""
    import lightzero_b200 as lzb
    from oracle import build_gmz_ref
    gref = build_gmz_ref.load()
    if gref is None:
        pytest.skip("compiled reference Gumbel tree not built (oracle/build_gmz_ref.py)")
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


@pytest.mark.parametrize("name", ["pendulum", "mountain_car"])
def test_collect_equals_initial_inference_prepare_and_search(name):
    import lightzero_b200 as lzb
    from lightzero_b200.collect import MuZeroCollectPolicy
    B, S = 16, 25
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


@pytest.mark.parametrize("name", ["pendulum", "mountain_car"])
def test_reanalyze_equals_its_manual_restatement(name):
    """one compute_target_policy_reanalyzed call against initial_inference + prepare + search + the target assembly"""
    import lightzero_b200 as lzb
    from lightzero_b200.reanalyze import compute_target_policy_reanalyzed
    segments, unroll, S = 6, 5, 16
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


# the model= dicts of the reference configs (zoo/...), with the keys the shipped configs pass
REFERENCE_DICTS = {
    "cartpole": dict(observation_shape=4, action_space_size=2, model_type='mlp', lstm_hidden_size=128, latent_state_dim=128,
                     self_supervised_learning_loss=True, discrete_action_encoding_type='one_hot', norm_type='BN'),
    "mountain_car": dict(observation_shape=2, action_space_size=3, model_type='mlp', lstm_hidden_size=128, latent_state_dim=64,
                         self_supervised_learning_loss=True, discrete_action_encoding_type='one_hot', norm_type='BN'),
    "pendulum": dict(observation_shape=3, action_space_size=11, model_type='mlp', lstm_hidden_size=128, latent_state_dim=128,
                     self_supervised_learning_loss=True),
    "bsuite_bandit": dict(observation_shape=1, action_space_size=11, model_type='mlp', lstm_hidden_size=128, latent_state_dim=128,
                          self_supervised_learning_loss=True, discrete_action_encoding_type='one_hot', norm_type='BN'),
    "bsuite_swingup": dict(observation_shape=8, action_space_size=3, model_type='mlp', lstm_hidden_size=128, latent_state_dim=128,
                           self_supervised_learning_loss=True, discrete_action_encoding_type='one_hot', norm_type='BN'),
    "memory": dict(analysis_sim_norm=False, observation_shape=25, action_space_size=4, model_type='mlp', latent_state_dim=128,
                   discrete_action_encoding_type='one_hot', norm_type='BN', self_supervised_learning_loss=True),
}


@pytest.mark.parametrize("name", list(REFERENCE_DICTS))
def test_reference_config_constructs_loads_and_searches(name):
    """the reference config's model dict as keywords, and a state_dict with the SSL heads it builds: ignored at inference.
    cartpole's dict has no res_connection_in_dynamics: it runs fc_dynamics, where the table's cartpole row runs the residual."""
    import lightzero_b200 as lzb
    kw = REFERENCE_DICTS[name]
    obs_dim, A, L = kw["observation_shape"], kw["action_space_size"], kw["latent_state_dim"]
    from oracle.model_ref import MuZeroModelMLPRef, emulate_trained_mlp_
    torch.manual_seed(1)
    ref = emulate_trained_mlp_(MuZeroModelMLPRef(obs_dim, A, L, res_connection_in_dynamics=False), 1)
    sd = dict(ref.state_dict())
    sd.update({"projection.0.weight": torch.randn(1024, L), "projection.1.running_mean": torch.randn(1024),
               "prediction_head.0.weight": torch.randn(512, 1024)})
    cu = lzb.MuZeroModelMLP(**kw).load_state_dict(sd)
    B, S = 8, 25
    obs = torch.rand(B, obs_dim) * 2 - 1
    action = torch.arange(B) % A
    out = cu.initial_inference(obs.cuda())
    with torch.no_grad():
        e0 = ref.initial_inference(obs)
        e1 = ref.recurrent_inference(e0.latent_state, action)
    close(out.latent_state, e0.latent_state, "latent")
    close(out.policy_logits, e0.policy_logits, "policy")
    o1 = cu.recurrent_inference(e0.latent_state.cuda(), action.cuda())
    close(o1.latent_state, e1.latent_state, "next latent")
    close(o1.reward, e1.reward, "reward logits")
    mcts = lzb.MuZeroMCTSCtree(dict(num_simulations=S))
    roots = mcts.roots(B, [list(range(A))] * B)
    roots.prepare_no_noise([0.] * B, out.policy_logits, [-1] * B)
    mcts.search(roots, cu, out.latent_state, [-1] * B)
    assert all(sum(d) == S for d in roots.get_distributions())
    roots.clear()


@pytest.mark.parametrize("name", NAMES)
def test_table_config_stays_on_the_fp32_kernels(name):
    from lightzero_b200 import cabi
    _, cu = make(name, 0)
    assert cu.value_support_size == len(torch.arange(*MR.CONFIGS[name][5]))
    with pytest.raises(cabi.LzError, match="no math mode"):
        cu.set_math("tc3")


def test_first_configs_past_each_edge_leave_the_fp32_kernels():
    """one step past each edge of the fp32 envelope: the tensor-core kernel takes it (a math mode exists) or nothing does"""
    import lightzero_b200 as lzb
    from lightzero_b200 import cabi
    base = dict(observation_shape=4, action_space_size=2, latent_state_dim=128)
    for kw in (dict(observation_shape=161), dict(action_space_size=33)):
        lzb.MuZeroModelMLP(**dict(base, **kw)).set_math("tc1").set_math("tc3")       # kind 4
    for kw, msg in ((dict(latent_state_dim=129), "latent_dim 129, obs_dim 4, action_space_size 2,"),
                    (dict(latent_state_dim=7), "latent_dim 7, obs_dim 4, action_space_size 2,"),
                    (dict(reward_head_hidden_channels=[161]), "head hidden sizes 161 / 32 / 32 fit neither"),
                    (dict(value_head_hidden_channels=[161]), "head hidden sizes 32 / 161 / 32 fit neither"),
                    (dict(policy_head_hidden_channels=[161]), "head hidden sizes 32 / 32 / 161 fit neither"),
                    (dict(latent_state_dim=100, action_space_size=61), "latent_dim 100, obs_dim 4, action_space_size 61,")):
        with pytest.raises(cabi.LzError, match=msg) as e:
            lzb.MuZeroModelMLP(**dict(base, **kw))
        assert "fit neither" in str(e.value)
    ok = lzb.MuZeroModelMLP(**dict(base, reward_support_range=(-303., 305., 1.), value_support_range=(-303., 305., 1.)))
    assert ok.value_support_size == 608
    with pytest.raises(cabi.LzError, match=r"support size 609 not in \[2, 608\]"):
        lzb.MuZeroModelMLP(**dict(base, reward_support_range=(-304., 305., 1.), value_support_range=(-304., 305., 1.)))


@pytest.mark.parametrize("head", ["fc_value_head", "fc_policy_head"])
def test_head_with_two_hidden_layers_is_refused_at_finalize(head):
    """the kernels run one hidden layer per head: a state_dict with two is refused, not packed"""
    import lightzero_b200 as lzb
    from lightzero_b200 import cabi
    from oracle.model_ref import MLP_V2_general
    ref = MR.build("pendulum", 0)
    L, A, K = 128, 11, 601
    deep = MLP_V2_general(L, [32, 32], K if head == "fc_value_head" else A, torch.nn.ReLU, False, False, False)
    setattr(ref.prediction_network, head, deep)
    cu = lzb.MuZeroModelMLP(**MR.model_kwargs("pendulum"))
    with pytest.raises(cabi.LzError, match=rf"tensor 'prediction_network\.{head}\.3\.(weight|bias)' has (1024|32) elements"):
        cu.load_state_dict(ref.state_dict())
