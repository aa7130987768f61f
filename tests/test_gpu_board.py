"""The board-game MuZero network (downsample=False, csrc/board_tc.cu) on the GPU.

- the CUDA model against the fixtures of the reference class and against the PyTorch restatement, both programs, at batch
  sizes that hit every CTA packing, a partial last CTA and a second wave (the launch plan is printed from the debug hook);
- one root's outputs are the same bits whatever its slot and packing;
- the fused searches (multi-kernel graph, search_with_reuse, Gumbel, lz_search_collect) against the oracle driving the same
  network, bit for bit;
- refusals of configurations outside the board kernel's space.
"""
import os

import numpy as np
import pytest
import torch

import board_model_ref as BR
from conftest import ROOT
from oracle import model_ref as R
from oracle.tree_drive import assert_same, drive, network, readout
from test_gpu_search_oracle import _inputs, fused_search, oracle_search, visits_sum_to, zero_policy

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(ROOT, "tests", "golden")
NAMES = list(BR.BOARD_CONFIGS)
BATCHES = (1, 2, 3, 7, 8, 9, 31, 32, 33, 129, 1024, 1201)
TOL = dict(rtol=1e-5, atol=1e-5)
TOL_SCALAR = dict(rtol=2e-4, atol=2e-4)


def make(name, seed=0, mutate=None, math="tc3"):
    import lightzero_b200 as lzb
    ref = BR.build(name, seed)
    if mutate is not None:
        mutate(ref)
    cu = lzb.MuZeroModel(**BR.model_kwargs(name)).load_state_dict(ref.state_dict())
    cu.set_math(math)
    return ref, cu


def support(name):
    return R.DiscreteSupport(*BR.BOARD_CONFIGS[name][6])


def scalar(logits, name):
    return R.inverse_scalar_transform(logits, support(name)).reshape(-1)


def plan(cu, which, B, x, action):
    """the launch plan of the program (lz_model_debug_net_stage at its last stage): R, NT, CTAs, roots of the last CTA"""
    from lightzero_b200 import cabi
    nres, A, K = BR.BOARD_CONFIGS[cu._name][3], cu.action_space_size, cu.value_support_size
    out = torch.empty(B * (2 * K + 2 * A + 4), device=cu.device)
    info = np.zeros(8, np.int32)
    with torch.cuda.device(cu.device):
        cabi.check(cu._lib.lz_model_debug_net_stage(cu._h, which, B, x.data_ptr(), cabi.ptr(action), 1 + 4 * nres, out.data_ptr(),
                                                    out.numel() * 4, info.ctypes.data, cabi.stream_ptr()), "lz_model_debug_net_stage")
    torch.cuda.synchronize()
    return dict(zip(("R", "NT", "ctas", "last", "layers", "npass", "smem"), (int(v) for v in info[:7])))


def close(got, exp, what, **tol):
    got, exp = got.detach().float().cpu(), exp.detach().float().cpu()
    assert got.shape == exp.shape, (what, got.shape, exp.shape)
    assert torch.allclose(got, exp, **tol), (what, float((got - exp).abs().max()))


@pytest.mark.parametrize("name", NAMES)
def test_model_against_fixture(name):
    d = np.load(os.path.join(GOLDEN, f"board_{name}.npz"))
    ref, cu = make(name, int(d["seed"]))
    obs, action = torch.from_numpy(d["obs"]), torch.from_numpy(d["action"])
    o0 = cu.initial_inference(obs.cuda(), return_scalar_value=True)
    assert tuple(o0.latent_state.shape) == (obs.shape[0], BR.BOARD_CONFIGS[name][2]) + tuple(obs.shape[2:])
    close(o0.latent_state, torch.from_numpy(d["init_latent_state"]), "init latent", **TOL)
    close(o0.policy_logits, torch.from_numpy(d["init_policy_logits"]), "init policy", **TOL)
    close(o0.value, torch.from_numpy(d["init_value"]), "init value logits", **TOL)
    close(o0.value_scalar, scalar(torch.from_numpy(d["init_value"]), name), "init value", **TOL_SCALAR)
    o1 = cu.recurrent_inference(torch.from_numpy(d["init_latent_state"]).cuda(), action.cuda(), return_scalars=True)
    for f in ("latent_state", "reward", "value", "policy_logits"):
        close(getattr(o1, f), torch.from_numpy(d["rec_" + f]), "rec " + f, **TOL)
    close(o1.reward_scalar, scalar(torch.from_numpy(d["rec_reward"]), name), "rec reward", **TOL_SCALAR)
    close(o1.value_scalar, scalar(torch.from_numpy(d["rec_value"]), name), "rec value", **TOL_SCALAR)


@pytest.mark.parametrize("name", NAMES)
def test_model_against_restatement_at_every_packing(name):
    ref, cu = make(name, 3)
    cu._name = name
    obs_shape, A = BR.BOARD_CONFIGS[name][0], BR.BOARD_CONFIGS[name][1]
    g = torch.Generator().manual_seed(7)
    plans = []
    for B in BATCHES:
        obs = torch.rand((B,) + tuple(obs_shape), generator=g)
        action = torch.randint(0, A, (B,), generator=g)
        with torch.no_grad():
            e0 = ref.initial_inference(obs)
            e1 = ref.recurrent_inference(e0.latent_state, action)
        o0 = cu.initial_inference(obs.cuda(), return_scalar_value=True)
        close(o0.latent_state, e0.latent_state, f"B={B} init latent", **TOL)
        close(o0.policy_logits, e0.policy_logits, f"B={B} init policy", **TOL)
        close(o0.value, e0.value, f"B={B} init value logits", **TOL)
        close(o0.value_scalar, scalar(e0.value, name), f"B={B} init value", **TOL_SCALAR)
        lat = e0.latent_state.cuda()
        a = action.to(torch.int32).cuda()
        o1 = cu.recurrent_inference(lat, a, return_scalars=True)
        for f in ("latent_state", "reward", "value", "policy_logits"):
            close(getattr(o1, f), getattr(e1, f), f"B={B} rec {f}", **TOL)
        close(o1.reward_scalar, scalar(e1.reward, name), f"B={B} rec reward", **TOL_SCALAR)
        close(o1.value_scalar, scalar(e1.value, name), f"B={B} rec value", **TOL_SCALAR)
        for which, x, act in ((0, lat, a), (1, obs.cuda().contiguous(), None)):
            p = plan(cu, which, B, x, act)
            assert p["ctas"] * p["R"] >= B > (p["ctas"] - 1) * p["R"] and p["last"] == B - (p["ctas"] - 1) * p["R"]
            assert (p["R"], p["NT"], p["ctas"], p["last"]) == BR.board_plan(BR.BOARD_CONFIGS[name][2], *obs_shape[1:], B), (B, p)
            plans.append((B, which, p["R"], p["NT"], p["ctas"], p["last"]))
    print(f"\n[board] {name} plans (B, program, R, NT, ctas, last): {plans}")
    assert any(p[5] != p[2] for p in plans)               # some launch ends in a partial CTA
    if name in ("connect4", "board8x8_r3", "board8x8_hc16"):
        assert any(p[4] > 132 for p in plans)              # and, with few roots per CTA, some runs a second wave


@pytest.mark.parametrize("name", NAMES)
def test_one_root_is_the_same_bits_at_every_slot(name):
    _, cu = make(name, 5)
    obs_shape, A = BR.BOARD_CONFIGS[name][0], BR.BOARD_CONFIGS[name][1]
    g = torch.Generator().manual_seed(11)
    one = torch.rand((1,) + tuple(obs_shape), generator=g)
    ref0 = cu.initial_inference(one.cuda(), return_scalar_value=True)
    ref1 = cu.recurrent_inference(ref0.latent_state, torch.tensor([A - 1], dtype=torch.int32).cuda(), return_scalars=True)
    for B in (2, 9, 33, 300):
        o0 = cu.initial_inference(one.expand((B,) + tuple(obs_shape)).contiguous().cuda(), return_scalar_value=True)
        o1 = cu.recurrent_inference(o0.latent_state, torch.full((B,), A - 1, dtype=torch.int32).cuda(), return_scalars=True)
        for got, exp in ((o0.latent_state, ref0.latent_state), (o0.policy_logits, ref0.policy_logits), (o0.value_scalar, ref0.value_scalar),
                         (o1.latent_state, ref1.latent_state), (o1.reward, ref1.reward), (o1.value, ref1.value),
                         (o1.policy_logits, ref1.policy_logits), (o1.reward_scalar, ref1.reward_scalar), (o1.value_scalar, ref1.value_scalar)):
            assert torch.equal(got.cpu(), exp.cpu().expand_as(got.cpu())), B


# name: config, B, S, deterministic, players, mutate, discount
SEARCHES = {
    "tictactoe_b8_s25_det_2p": ("tictactoe", 8, 25, True, "2p", None, 1.0),
    "tictactoe_b32_s30_sto_zero_policy_2p": ("tictactoe", 32, 30, False, "2p", zero_policy, 1.0),
    "tictactoe_b9_s25_det_1p": ("tictactoe", 9, 25, True, "1p", None, 0.997),
    "gomoku_b32_s50_sto_2p": ("gomoku", 32, 50, False, "2p", None, 1.0),
    "connect4_b8_s50_det_mixed": ("connect4", 8, 50, True, "mixed", None, 1.0),
    "board8x8_b40_s20_sto_mixed": ("board8x8_r3", 40, 20, False, "mixed", None, 1.0),
    # each channel width at its largest tile count, where the leaves' latents are gathered for many roots per CTA
    "board8x8_hc16_b661_s6_det_mixed": ("board8x8_hc16", 661, 6, True, "mixed", None, 0.997),     # C16 NT8: 6 roots per CTA
    "gomoku_b1201_s6_det_2p": ("gomoku", 1201, 6, True, "2p", None, 1.0),                          # C32 NT8: 10 roots per CTA
    "board8x8_b300_s6_det_2p": ("board8x8_r3", 300, 6, True, "2p", None, 1.0),                      # C64 NT4: 3 roots per CTA
}
WIDEST = {"board8x8_hc16_b661_s6_det_mixed": 8, "gomoku_b1201_s6_det_2p": 8, "board8x8_b300_s6_det_2p": 4}


@pytest.mark.parametrize("case", list(SEARCHES))
def test_fused_search_equals_oracle_driving_the_same_network(case):
    import lightzero_b200 as lzb
    name, B, S, det, players, mutate, disc = SEARCHES[case]
    _, cu = make(name, 2, mutate)
    A = cu.action_space_size
    seed = sum(map(ord, case))
    obs = torch.rand((B,) + tuple(BR.BOARD_CONFIGS[name][0]), generator=torch.Generator().manual_seed(seed))
    latent = cu.initial_inference(obs.cuda()).latent_state
    legal, logits, noises, tp = _inputs(B, A, seed, players)
    if players == "2p":                                    # players alternate along the batch
        tp = [1 + b % 2 for b in range(B)]
    mcts = lzb.MuZeroMCTSCtree(dict(num_simulations=S, deterministic=det, discount_factor=disc))
    got, key, plan_, roots = fused_search(cu, mcts, S, latent, legal, logits, noises, tp)
    exp, st = oracle_search(cu, S, latent, legal, logits, noises, tp, det, key=key, discount=disc)
    kernels = mcts.last_num_kernels
    roots.clear()
    R, NT = BR.board_plan(BR.BOARD_CONFIGS[name][2], *BR.BOARD_CONFIGS[name][0][1:], B)[:2]
    print(f"\n[board-search] {case}: ties={st['ties']} draws={st['draws']} kernels={kernels} R={R} NT={NT}")
    assert NT == WIDEST.get(case, NT)
    assert_same(got, exp)
    assert visits_sum_to(got, S)
    assert not plan_["persistent"] and kernels == 2 * S + 1    # the multi-kernel search graph
    assert min(len(l) for l in legal) == 1                     # a root with a single legal action
    if not det:
        assert st["ties"] > 0 and st["draws"] > 0


@pytest.mark.parametrize("name", ["connect4", "gomoku"])
def test_search_with_reuse_equals_stepwise_drive(name):
    import lightzero_b200 as lzb
    from lightzero_b200 import mz_tree
    B, S = 24, 30
    _, cu = make(name, 4)
    A = cu.action_space_size
    obs = torch.rand((B,) + tuple(BR.BOARD_CONFIGS[name][0]), generator=torch.Generator().manual_seed(4))
    out = cu.initial_inference(obs.cuda())
    legal, _, noises, tp = _inputs(B, A, 9, "2p")
    rng = np.random.default_rng(3)
    true_action = [int(l[rng.integers(len(l))]) for l in legal]
    reuse_value = (rng.standard_normal(B) * 0.5).astype(np.float32).tolist()
    mcts = lzb.MuZeroMCTSCtree(dict(num_simulations=S, deterministic=True, discount_factor=1.0))
    roots = mcts.roots(B, legal)
    roots.prepare(0.25, noises, [0.] * B, out.policy_logits, tp)
    mcts.search_with_reuse(roots, cu, out.latent_state, tp, true_action, reuse_value)
    fused = readout(roots, A, S)
    roots.clear()
    c = dict(B=B, A=A, S=S, legal=legal, root_logits=out.policy_logits.cpu().numpy(), noises=noises, to_play=tp,
             true_action=true_action, reuse_value=reuse_value, discount=1.0)
    step, _ = drive(mz_tree, c, "reuse", network(cu, out.latent_state))
    assert_same(step, fused)
    assert min(step["n_inferred"].tolist()) < B


@pytest.mark.parametrize("name", ["tictactoe", "gomoku"])
def test_gumbel_search_equals_reference_tree(name):
    import lightzero_b200 as lzb
    from oracle import build_gmz_ref
    gref = build_gmz_ref.load()
    if gref is None:
        pytest.skip("compiled reference Gumbel tree not built")
    B, S, m = 16, 16, 4
    _, cu = make(name, 6)
    A = cu.action_space_size
    obs = torch.rand((B,) + tuple(BR.BOARD_CONFIGS[name][0]), generator=torch.Generator().manual_seed(6))
    out = cu.initial_inference(obs.cuda(), return_scalar_value=True)
    legal, _, noises, tp = _inputs(B, A, 12, "1p", masks=False)
    gmcts = lzb.GumbelMuZeroMCTSCtree(dict(num_simulations=S, max_num_considered_actions=m))
    roots = gmcts.roots(B, legal)
    roots.prepare(0.25, noises, [0.] * B, out.value_scalar, out.policy_logits, tp)
    gmcts.search(roots, cu, out.latent_state, tp)
    dist, vals, pol = roots.get_distributions(), roots.get_values(), roots.get_policies(0.997, A)
    roots.clear()
    c = dict(B=B, A=A, S=S, legal=legal, root_logits=out.policy_logits.cpu().numpy(), noises=noises, to_play=tp, m=m,
             root_values=out.value_scalar.cpu().numpy())
    t, _ = drive(gref, c, "gumbel", network(cu, out.latent_state))
    assert t["distributions"].tolist() == dist
    assert np.array_equal(t["root_values_bits"], np.asarray(vals, np.float32).view(np.uint32))
    assert np.array_equal(t["policies"].view(np.uint32), np.asarray(pol, np.float32).view(np.uint32))


def test_collect_equals_initial_inference_prepare_and_search():
    import lightzero_b200 as lzb
    from lightzero_b200.collect import MuZeroCollectPolicy
    name, B, S = "connect4", 16, 25
    _, cu = make(name, 8)
    A = cu.action_space_size
    obs = torch.rand((B,) + tuple(BR.BOARD_CONFIGS[name][0]), generator=torch.Generator().manual_seed(8))
    legal, _, noises, tp = _inputs(B, A, 13, "2p")
    mask = np.zeros((B, A), np.uint8)
    for b, l in enumerate(legal):
        mask[b, l] = 1
    noise_rows = np.zeros((B, A), np.float32)
    for b, n in enumerate(noises):
        noise_rows[b, :len(n)] = n
    pol = MuZeroCollectPolicy(cu, dict(num_simulations=S, deterministic=True, discount_factor=1.0))
    got = pol.search_batch(obs.cuda(), mask, noise_rows, tp, read_back=False)
    out = cu.initial_inference(obs.cuda(), return_scalar_value=True)
    mcts = lzb.MuZeroMCTSCtree(dict(num_simulations=S, deterministic=True, discount_factor=1.0))
    roots = mcts.roots(B, legal)
    roots.prepare(0.25, noises, [0.] * B, out.policy_logits, tp)
    mcts.search(roots, cu, out.latent_state, tp)
    exp = readout(roots, A, S)
    roots.clear()
    assert torch.equal(got["pred_value"].cpu(), out.value_scalar.cpu())
    assert torch.equal(got["policy_logits"].cpu(), out.policy_logits.cpu())
    visits = got["visits"].cpu().numpy()
    assert np.array_equal(visits, exp["distributions"])
    assert np.array_equal(got["values"].cpu().numpy().view(np.uint32), exp["root_values_bits"])


def test_refusals():
    import lightzero_b200 as lzb
    from lightzero_b200 import cabi
    for shape in ((3, 9, 9), (3, 15, 15)):
        with pytest.raises(NotImplementedError, match="downsample"):
            lzb.MuZeroModel(observation_shape=shape, action_space_size=shape[1] * shape[2], downsample=False)
    with pytest.raises(cabi.LzError, match="num_channels"):
        lzb.MuZeroModel(observation_shape=(3, 6, 6), action_space_size=36, num_channels=48)
    with pytest.raises(cabi.LzError, match="observation planes"):
        lzb.MuZeroModel(observation_shape=(17, 6, 6), action_space_size=36, num_channels=32)
    with pytest.raises(NotImplementedError, match="downsample"):
        lzb.EfficientZeroModel(observation_shape=(3, 3, 3), action_space_size=9, downsample=False)
    # one step outside each corner of row1x8_r4, col8x1 and board8x8_hc16
    for kw, msg in ((dict(action_space_size=65), "1 to 64 actions"), (dict(num_res_blocks=5), "num_res_blocks"),
                    (dict(reward_head_channels=17), "head channels"), (dict(policy_head_channels=0), "head channels"),
                    (dict(value_head_channels=0), "head channels"), (dict(value_head_hidden_channels=[33]), "hidden sizes"),
                    (dict(reward_head_hidden_channels=[0]), "hidden sizes"), (dict(policy_head_hidden_channels=[0]), "hidden sizes")):
        with pytest.raises(cabi.LzError, match=msg):
            lzb.MuZeroModel(**dict(BR.model_kwargs("board8x8_hc16"), **kw))
    # uint8 frames are the Atari path: a board model refuses them
    _, cu = make("tictactoe", 1)
    mcts = lzb.MuZeroMCTSCtree(dict(num_simulations=4))
    roots = mcts.roots(2, [list(range(9))] * 2)
    roots.prepare_no_noise([0.] * 2, np.zeros((2, 9), np.float32), [-1, -1])
    roots._materialize(4)
    t = roots._tree
    q = t.search_for(cu, 4)
    frames = torch.zeros(2, 3, 3, 3, dtype=torch.uint8, device="cuda")
    rc = cu._lib.lz_search_collect_u8(q, frames.data_ptr(), None, None, 0.0, None, 1, None, None, cabi.stream_ptr())
    assert rc == -1 and b"conv model" in cu._lib.lz_last_error()
    roots.clear()
