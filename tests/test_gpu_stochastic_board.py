"""GPU tests of Stochastic MuZero on board observations (StochasticMuZeroModel with downsample=False, the 2048 network, on the
board tensor-core kernel):
- the model: initial_inference and both recurrent programs against the reference class's fixtures, and against the float64
  restatement at batch sizes that give every (R, NT) launch plan of each config with a partial last CTA; one root repeated over
  a whole launch gives the same bits at every row;
- masked launches of both recurrent programs: selected rows equal the unmasked launch bit for bit, every other row keeps a
  sentinel in every output (an all-zero mask, and zeros covering whole CTAs);
- the fused search equals the compiled reference tree driving the same CUDA network, bit for bit, with the chance draw pinned
  (one and two players, masked legal actions, chance > A and A > chance, 2048 at B = 8 and 256 with S = 100); a sampled
  search repeats bit for bit for one RNG key;
- the collect step equals initial_inference + prepare + search; SegmentStats keeps the first A columns; the buffer's value
  targets equal oracle/targets_ref.py; the collect on a side stream; one captured graph per shape;
- refusals: downsample=True, a MuZero tree with the stochastic model and the reverse, the reuse search on a stochastic tree,
  lz_model_create_stochastic outside its envelope."""
import os
import sys

import numpy as np
import pytest
import torch

import stoch_board_model_ref as SB
from conftest import ROOT
from test_gpu_stochastic import assert_equal, close, readout, reference_loop, scalar
from test_gpu_streams import _check_on_side_stream, sleep_rate  # noqa: F401  (the streams harness and its fixture)

pytestmark = pytest.mark.gpu

NAMES = list(SB.CONFIGS)
GOLDEN = os.path.join(ROOT, "tests", "golden")
if GOLDEN not in sys.path:
    sys.path.insert(0, GOLDEN)      # make_model_golden.weights_digest
DISCOUNT = 0.997
_models = {}


def model(name):
    """(float32 restatement, CUDA StochasticMuZeroModel) of a config with the fixture's weights, one per config"""
    import lightzero_b200 as lzb
    if name not in _models:
        ref = SB.build(name, NAMES.index(name))
        sd = dict(ref.state_dict())
        sd["chance_encoder.encoder.conv1.weight"] = torch.randn(4, 4)      # training-only keys ride along and are ignored
        _models[name] = ref, lzb.StochasticMuZeroModel(**SB.model_kwargs(name)).load_state_dict(sd)
    return _models[name]


def plans(name):
    """{R: B} with B = 132 R - 1: R roots per CTA (every NT the plan picks), the last CTA one root short when R > 1"""
    C, (_, H, W) = SB.CONFIGS[name][3], SB.CONFIGS[name][0]
    rpr, pad = (H + 1) * (W + 1), W + 2
    rmax = max(1, ((4 if C == 64 else 8) * 64 + pad) // rpr)
    return {R: 132 * R - 1 for R in range(1, rmax + 1)}


def rand_inputs(name, B, seed):
    obs_shape, A, NC = SB.CONFIGS[name][:3]
    g = torch.Generator().manual_seed(seed)
    return (torch.rand((B,) + tuple(obs_shape), generator=g), torch.randint(0, A, (B,), generator=g),
            torch.randint(0, NC, (B,), generator=g))


# ---- the model -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", NAMES)
def test_model_matches_fixture(name):
    from make_model_golden import weights_digest
    ref, cu = model(name)
    z = np.load(os.path.join(GOLDEN, f"stoch_board_{name}.npz"))
    assert str(z["weights_sha256"]) == weights_digest(ref)      # the fixture was made from these weights
    sup = SB.CONFIGS[name][7]
    o = cu.initial_inference(torch.from_numpy(z["obs"]).cuda(), return_scalar_value=True)
    for f in ("value", "policy_logits", "latent_state"):
        close(getattr(o, f).cpu(), z["init_" + f], f"{name} initial {f}")
    close(o.value_scalar.cpu(), scalar(z["init_value"], sup), f"{name} initial value", 2e-4)
    a = cu.recurrent_inference(torch.from_numpy(z["init_latent_state"]).cuda(), torch.from_numpy(z["action"]).cuda(), False,
                               return_scalars=True)
    r = cu.recurrent_inference(torch.from_numpy(z["after_latent_state"]).cuda(), torch.from_numpy(z["chance"]).cuda(), True,
                               return_scalars=True)
    for prefix, got in (("after_", a), ("rec_", r)):
        for f in ("value", "reward", "policy_logits", "latent_state"):
            close(getattr(got, f).cpu(), z[prefix + f], f"{name} {prefix}{f}")
        close(got.value_scalar.cpu(), scalar(z[prefix + "value"], sup), f"{name} {prefix}value", 2e-4)
        close(got.reward_scalar.cpu(), scalar(z[prefix + "reward"], sup), f"{name} {prefix}reward", 2e-4)
    assert a.policy_logits.shape == (5, cu.chance_space_size) and r.policy_logits.shape == (5, cu.action_space_size)


@pytest.mark.parametrize("name", NAMES)
def test_model_float64_at_every_packing(name):
    ref, cu = model(name)
    ref64 = SB.build(name, NAMES.index(name), torch.float64).cuda()
    sup = SB.CONFIGS[name][7]
    for R, B in plans(name).items():
        obs, act, ch = (x.cuda() for x in rand_inputs(name, B, B))
        o = cu.initial_inference(obs, return_scalar_value=True)
        with torch.no_grad():
            e0 = ref64.initial_inference(obs.double())
            ea = ref64.recurrent_inference(o.latent_state.double(), act, False)
            er = ref64.recurrent_inference(ea.latent_state.float().double(), ch, True)
        close(o.latent_state.cpu(), e0.latent_state.cpu(), f"R={R} initial latent")
        close(o.policy_logits.cpu(), e0.policy_logits.cpu(), f"R={R} initial policy")
        close(o.value_scalar.cpu(), scalar(e0.value.cpu(), sup), f"R={R} initial value", 2e-4)
        a = cu.recurrent_inference(o.latent_state, act, False, return_scalars=True)
        r = cu.recurrent_inference(ea.latent_state.float(), ch, True, return_scalars=True)
        for what, got, exp in (("afterstate", a, ea), ("dynamics", r, er)):
            for f in ("latent_state", "policy_logits", "value", "reward"):
                close(getattr(got, f).cpu(), getattr(exp, f).cpu(), f"R={R} {what} {f}")
            close(got.value_scalar.cpu(), scalar(exp.value.cpu(), sup), f"R={R} {what} value", 2e-4)
            close(got.reward_scalar.cpu(), scalar(exp.reward.cpu(), sup), f"R={R} {what} reward", 2e-4)


@pytest.mark.parametrize("name", ["game_2048", "c16_3x3_ch1", "c32_6x7_ch20"])
def test_one_root_same_bits_at_every_row(name):
    """one root repeated over a launch of the largest R: every row of every program's outputs has the bits of row 0"""
    _, cu = model(name)
    B = max(plans(name).values())
    obs, act, ch = (x[:1].cuda() for x in rand_inputs(name, 1, 5))
    o = cu.initial_inference(obs.expand((B,) + tuple(obs.shape[1:])).contiguous(), return_scalar_value=True)
    a = cu.recurrent_inference(o.latent_state, act.expand(B), False, return_scalars=True)
    r = cu.recurrent_inference(a.latent_state, ch.expand(B), True, return_scalars=True)
    for what, out, fields in (("initial", o, ("latent_state", "policy_logits", "value", "value_scalar")),
                              ("afterstate", a, ("latent_state", "policy_logits", "value", "reward", "value_scalar", "reward_scalar")),
                              ("dynamics", r, ("latent_state", "policy_logits", "value", "reward", "value_scalar", "reward_scalar"))):
        for f in fields:
            x = getattr(out, f)
            assert torch.equal(x, x[:1].expand_as(x)), (what, f)


@pytest.mark.parametrize("afterstate", [False, True])
@pytest.mark.parametrize("mask_kind", ["random", "zero"])
def test_masked_launch(afterstate, mask_kind):
    from lightzero_b200 import cabi
    _, cu = model("game_2048")
    A, NC, K = cu.action_space_size, cu.chance_space_size, cu.value_support_size
    B = 900                      # R = 7 roots per CTA
    g = torch.Generator().manual_seed(3)
    state = torch.rand((B,) + cu.latent_shape, generator=g).cuda()
    opt = torch.randint(0, NC if afterstate else A, (B,), generator=g).int().cuda()
    mask = torch.randint(0, 4, (B,), generator=g).int().cuda()
    mask[7:21] = 0               # CTAs 1 and 2 have no selected root
    if mask_kind == "zero":
        mask.zero_()
    full = cu.recurrent_inference(state, opt, afterstate, return_scalars=True)
    P = A if afterstate else NC
    outs = [torch.full(s, 7.25, device="cuda") for s in ((B,) + cu.latent_shape, (B, K), (B, K), (B, P), (B,), (B,))]
    cabi.check(cu._lib.lz_model_recurrent_inference_stochastic(cu._h, int(afterstate), B, state.data_ptr(), opt.data_ptr(),
                                                               mask.data_ptr(), 1, *(o.data_ptr() for o in outs),
                                                               cabi.stream_ptr()), "masked")
    sel = (mask & 1) == 1
    exp = (full.latent_state, full.reward, full.value, full.policy_logits, full.reward_scalar, full.value_scalar)
    for got, e in zip(outs, exp):
        assert torch.equal(got[sel], e[sel])
        assert bool((got[~sel] == 7.25).all())


# ---- the search ----------------------------------------------------------------------------------------------------------
def case(name, B, two_player, masked, seed):
    _, cu = model(name)
    obs_shape, A = SB.CONFIGS[name][:2]
    rng = np.random.default_rng(seed)
    o = cu.initial_inference(torch.from_numpy(rng.random((B,) + tuple(obs_shape), dtype=np.float32)).cuda())
    legal = [sorted(rng.choice(A, rng.integers(1, A + 1), replace=False).tolist()) if masked else list(range(A))
             for _ in range(B)]
    noises = [rng.dirichlet([0.3] * len(l)).astype(np.float32).tolist() for l in legal]
    to_play = [int(x) for x in rng.integers(1, 3, B)] if two_player else [-1] * B
    return cu, o, legal, noises, to_play


SEARCH_CASES = [("game_2048", 8, False, True, 0, 100), ("game_2048", 256, False, False, 1, 100),
                ("game_2048", 256, True, True, 2, 100), ("c32_6x7_a12", 40, True, True, 3, 60),
                ("c32_6x7_ch20", 33, False, True, 4, 60)]


@pytest.mark.parametrize("name,B,two_player,masked,seed,S", SEARCH_CASES)
def test_fused_search_equals_reference_tree(name, B, two_player, masked, seed, S):
    from oracle import build_stoch_ref
    import lightzero_b200 as lzb
    oracle = build_stoch_ref.load()
    if oracle is None:
        pytest.skip("compiled reference Stochastic MuZero tree not built")
    cu, o, legal, noises, to_play = case(name, B, two_player, masked, seed)
    logits = o.policy_logits.cpu().tolist()
    chance_seed = 2000 + seed
    _, ref_roots = reference_loop(oracle, cu, o.latent_state, legal, logits, noises, to_play, S, chance_seed)
    want = readout(ref_roots)
    mcts = lzb.StochasticMuZeroMCTSCtree(dict(num_simulations=S, deterministic=True, chance_seed=chance_seed))
    roots = mcts.roots(B, legal, cu.chance_space_size)
    roots.prepare(0.25, noises, [0.] * B, logits, to_play)
    mcts.search(roots, cu, o.latent_state, to_play)
    assert mcts.last_num_kernels == 3 * S + 1
    assert_equal(readout(roots), want)
    assert all(sum(d) == S for d in readout(roots)["dist"])


def test_sampled_search_repeats():
    """chance_seed=None: the reference loop driving the device trees step by step and the fused search, on two fresh trees
    with one RNG key, draw the same chance outcomes: the sampled search repeats bit for bit"""
    import lightzero_b200 as lzb
    from lightzero_b200 import cabi, stochastic_mz_tree as T
    B, S = 53, 40                # a shape no other test pools: both trees are fresh
    cu, o, legal, noises, to_play = case("game_2048", B, False, True, 9)
    logits = o.policy_logits.cpu().tolist()
    _, step = reference_loop(T, cu, o.latent_state, legal, logits, noises, to_play, S, None)
    mcts = lzb.StochasticMuZeroMCTSCtree(dict(num_simulations=S, deterministic=True, chance_seed=None))
    fused = mcts.roots(B, legal, cu.chance_space_size)
    fused.prepare(0.25, noises, [0.] * B, logits, to_play)
    mcts.search(fused, cu, o.latent_state, to_play)
    assert fused._tree is not step._tree
    keys = []
    for r in (step, fused):
        seed, epoch, counter = (cabi.ctypes.c_uint64(), cabi.ctypes.c_uint64(), cabi.ctypes.c_uint32())
        cabi.check(r._tree.lib.lz_tree_debug_rng(r._tree.h, cabi.ctypes.byref(seed), cabi.ctypes.byref(epoch),
                                                 cabi.ctypes.byref(counter)), "lz_tree_debug_rng")
        keys.append((seed.value, epoch.value))
    assert keys[0] == keys[1]
    assert_equal(readout(fused), readout(step))


# ---- the collect ---------------------------------------------------------------------------------------------------------
def collect_inputs(name, B, masked, two_player, seed):
    """(obs f32 host, mask uint8 [B, A], noises f32 [B, A] in legal order, to_play int32 [B])"""
    obs_shape, A = SB.CONFIGS[name][:2]
    rng = np.random.default_rng(seed)
    obs = rng.random((B,) + tuple(obs_shape), dtype=np.float32)
    mask = np.ones((B, A), np.uint8)
    if masked:
        mask = (rng.random((B, A)) < 0.6).astype(np.uint8)
        mask[np.arange(B), rng.integers(0, A, B)] = 1
    noises = np.zeros((B, A), np.float32)
    for b in range(B):
        n = int(mask[b].sum())
        noises[b, :n] = rng.dirichlet([0.3] * n)
    to_play = rng.integers(1, 3, B).astype(np.int32) if two_player else np.full(B, -1, np.int32)
    return obs, mask, noises, to_play


def policy(cu, S, chance_seed):
    import lightzero_b200 as lzb
    return lzb.StochasticMuZeroCollectPolicy(cu, dict(num_simulations=S, deterministic=True, chance_seed=chance_seed,
                                                      discount_factor=DISCOUNT))


@pytest.mark.parametrize("name,B,masked,two_player", [("game_2048", 8, True, False), ("game_2048", 300, False, False),
                                                      ("c32_6x7_a12", 64, True, True)])
def test_collect_equals_stepwise(name, B, masked, two_player):
    from test_gpu_stochastic_collect import assert_same, stepwise
    _, cu = model(name)
    S = 50
    obs, mask, noises, to_play = collect_inputs(name, B, masked, two_player, B)
    exp = stepwise(cu, obs, mask, noises, to_play, S, 77)
    pol = policy(cu, S, 77)
    got = pol.search_batch(torch.from_numpy(obs).cuda(), torch.from_numpy(mask).cuda(), torch.from_numpy(noises).cuda(),
                           to_play, read_back=False)
    assert got["visits"].shape == (B, max(cu.action_space_size, cu.chance_space_size))
    assert_same(got, exp, cu.action_space_size)
    assert pol.last_num_kernels == 3 * S + 1


def test_segment_stats_store_first_a_columns():
    from lightzero_b200.collector import SegmentStats
    _, cu = model("game_2048")
    A = cu.action_space_size
    B, S, T = 8, 25, 3
    seg = SegmentStats(B, T, A)
    pol = policy(cu, S, 8)
    want = []
    for step in range(2):
        obs, mask, noises, to_play = collect_inputs("game_2048", B, True, False, 40 + step)
        r = pol.search_batch(torch.from_numpy(obs).cuda(), torch.from_numpy(mask).cuda(), torch.from_numpy(noises).cuda(),
                             to_play, read_back=False)
        seg.store_search_stats(r["visits"], r["values"])
        v = r["visits"][:, :A].cpu().numpy().astype(np.int64)
        assert (r["visits"][:, A:] == -1).all()
        pos = np.where(v > 0, v, 0)
        want.append(((pos / pos.sum(1, keepdims=True)).astype(np.float32), r["values"].cpu().numpy()))
    child, values, lens = seg.tensors()
    assert child.shape == (B, T, A)
    for t, (c, v) in enumerate(want):
        assert np.array_equal(child[:, t].cpu().numpy(), c)
        assert np.array_equal(values[:, t].cpu().numpy(), v)


@pytest.mark.parametrize("case_name", ["mz_f32_n7_k6", "mz_2p_f32_n64_k6"])
def test_value_targets(case_name):
    """the MuZero buffer's targets with the board stochastic model (its init program's values) equal oracle/targets_ref.py"""
    from oracle.targets_ref import reward_value_targets
    from lightzero_b200.reanalyze import compute_target_reward_value
    from value_targets_cases import CASES as VCASES, make_context, seed_of
    case_ = VCASES[case_name]
    _, cu = model("game_2048")
    seed = seed_of(case_name)
    ctx = make_context(case_, seed, cu.action_space_size)
    T = case_["N"] * case_["K1"]
    obs = torch.rand((T,) + cu.observation_shape, generator=torch.Generator().manual_seed(seed))
    args = (ctx["value_mask"], ctx["pos"], ctx["rewards_list"], ctx["game_segment_lens"], ctx["td_steps_list"],
            ctx["to_play_segment"])
    kw = dict(num_unroll_steps=case_["K1"] - 1, discount_factor=case_["discount"], env_type=ctx["env_type"])
    got = compute_target_reward_value(cu, obs, *args, mini_infer_size=40, return_values=True, **kw)
    values = torch.cat([cu.initial_inference(obs[b:b + 40].cuda(), return_scalar_value=True).value_scalar
                        for b in range(0, T, 40)]).cpu().numpy()
    assert np.array_equal(got[2].cpu().numpy().view(np.uint32), values.view(np.uint32))
    exp = reward_value_targets(values, *args, **kw)
    for a, b in zip(got[:2], exp[:2]):
        assert np.array_equal(a.view(np.uint64), np.asarray(b, np.float64).view(np.uint64))


def test_collect_on_side_stream(sleep_rate):
    """the collect step (initial_inference, reset, prepare and the fused search graph), model and trees created on a side
    stream next to a busy legacy default stream: no call waits for the default stream and the outputs equal a default-stream
    run bit for bit (tests/test_gpu_streams.py's harness)"""
    import lightzero_b200 as lzb
    name, B, S = "game_2048", 96, 25
    obs_shape, A = SB.CONFIGS[name][:2]
    sd = SB.build(name, NAMES.index(name)).state_dict()
    rng = np.random.default_rng(12)
    x = torch.from_numpy(rng.random((B,) + obs_shape, dtype=np.float32)).cuda()
    mask = torch.ones(B, A, dtype=torch.uint8, device="cuda")
    noises = torch.from_numpy(rng.dirichlet([0.3] * A, B).astype(np.float32)).cuda()

    def scenario():
        cu = lzb.StochasticMuZeroModel(**SB.model_kwargs(name)).load_state_dict(sd)
        pol = policy(cu, S, 17)
        r = pol.search_batch(x, mask, noises, [-1] * B, read_back=False)
        return dict({k: v.clone() for k, v in r.items()}, _keep=(cu, pol))
    _check_on_side_stream(sleep_rate, "stochastic board collect", scenario)


def test_one_graph_per_shape():
    """a repeated collect step replays the captured graph of 3S + 1 kernels: no new capture"""
    from lightzero_b200 import cabi
    _, cu = model("game_2048")
    B, S = 128, 25
    obs, mask, noises, to_play = collect_inputs("game_2048", B, True, False, 2)
    pol = policy(cu, S, None)
    x = torch.from_numpy(obs).cuda()
    pol.search_batch(x, mask, noises, to_play, read_back=False)
    lib = cabi.load()
    before = lib.lz_debug_graph_captures()
    for _ in range(3):
        pol.search_batch(x, mask, noises, to_play, read_back=False)
    torch.cuda.synchronize()
    assert lib.lz_debug_graph_captures() == before
    assert pol.last_num_kernels == 3 * S + 1


# ---- refusals ------------------------------------------------------------------------------------------------------------
def test_refusals():
    import lightzero_b200 as lzb
    import board_model_ref as BR
    from lightzero_b200 import cabi
    with pytest.raises(NotImplementedError, match="downsample=True"):
        lzb.StochasticMuZeroModel(observation_shape=(12, 96, 96), action_space_size=6, downsample=True)
    cu, o, legal, noises, to_play = case("game_2048", 8, False, False, 3)
    # a MuZero tree with the stochastic model
    mz = lzb.MuZeroMCTSCtree(dict(num_simulations=5))
    roots = mz.roots(8, legal)
    roots.prepare_no_noise([0.] * 8, o.policy_logits, to_play)
    with pytest.raises(cabi.LzError, match="stochastic mode"):
        mz.search(roots, cu, o.latent_state, to_play)
    # a stochastic tree (search graph and collect) with a MuZero board model
    board = lzb.MuZeroModel(**BR.model_kwargs("tictactoe")).load_state_dict(BR.build("tictactoe", 0).state_dict())
    st = lzb.StochasticMuZeroMCTSCtree(dict(num_simulations=5, chance_seed=1))
    sroots = st.roots(8, [list(range(9))] * 8, 2)
    sroots.prepare_no_noise([0.] * 8, torch.zeros(8, 9), to_play)
    sroots._materialize(5, st._params(), True)
    with pytest.raises(cabi.LzError, match="stochastic mode"):
        sroots._tree.search_for(board, 5)
    with pytest.raises(TypeError):
        lzb.StochasticMuZeroCollectPolicy(board, dict(num_simulations=5))
    # the reuse search on a stochastic tree
    mcts = lzb.StochasticMuZeroMCTSCtree(dict(num_simulations=5, chance_seed=1))
    r = mcts.roots(8, legal, cu.chance_space_size)
    r.prepare_no_noise([0.] * 8, o.policy_logits, to_play)
    mcts.search(r, cu, o.latent_state, to_play)
    with pytest.raises(NotImplementedError):
        mcts.search_with_reuse(r, cu, o.latent_state, to_play, [0] * 8, [0.] * 8)
    q = r._tree.search_for(cu, 5)
    ta, rv = torch.zeros(8, dtype=torch.int32, device="cuda"), torch.zeros(8, device="cuda")
    with pytest.raises(cabi.LzError, match="stochastic tree"):
        cabi.check(r._tree.lib.lz_search_run_with_reuse(q, o.latent_state.data_ptr(), None, None, ta.data_ptr(), rv.data_ptr(),
                                                        None, cabi.stream_ptr()), "lz_search_run_with_reuse")
    # lz_model_create_stochastic outside its envelope
    lib = cabi.load()
    ok = dict(obs_c=16, obs_h=4, obs_w=4, action_space_size=4, num_res_blocks=1, num_channels=64, reward_head_channels=16,
              value_head_channels=16, policy_head_channels=16, reward_hidden=32, value_hidden=32, policy_hidden=32,
              support_min=0., support_max=601., support_step=1., efficientzero=0, lstm_hidden_size=0, downsample=0)
    for change, chance, msg in ((dict(downsample=1), 32, "Atari Stochastic MuZero"), (dict(efficientzero=1), 32, "efficientzero"),
                                ({}, 0, "chance_space_size"), ({}, 65, "chance_space_size"),
                                (dict(num_channels=48), 32, "num_channels"), (dict(obs_h=9), 32, "boards up to"),
                                (dict(obs_c=17), 32, "observation planes"), (dict(action_space_size=65), 32, "actions")):
        cfg = cabi.StochasticConfig(cabi.ModelConfig(**dict(ok, **change)), chance)
        h = cabi.c_void_p()
        with pytest.raises(cabi.LzError, match=msg):
            cabi.check(lib.lz_model_create_stochastic(cfg, h), "lz_model_create_stochastic")
    h = cabi.c_void_p()
    cabi.check(lib.lz_model_create_stochastic(cabi.StochasticConfig(cabi.ModelConfig(**ok), 64), h), "inside the envelope")
    lib.lz_model_destroy(h)
