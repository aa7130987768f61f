"""The replay buffer's reward / value targets on the device (``reanalyze.compute_target_reward_value``, ``lz_value_targets`` /
``lz_value_targets_root``) bit for bit against oracle/targets_ref.py fed the same fp32 values.

The restatement is pinned to the reference's own _compute_target_reward_value by tests/test_value_targets_cpu.py.  Here it
bootstraps from the value scalars the CUDA model returns for the same observations (``initial_inference(...,
return_scalar_value=True)``) or, for EfficientZero's use_root_value, from the root values of the existing mirror pipeline
(``Roots.prepare`` + ``EfficientZeroMCTSCtree.search`` + ``get_values``).  Contexts come from the case grid of
tests/value_targets_cases.py.
"""
import numpy as np
import pytest
import torch

from oracle.targets_ref import reward_value_targets
from test_gpu_rezero_reanalyze import _conv_sd, make_model as rezero_model
from value_targets_cases import CASES, make_context, seed_of

pytestmark = pytest.mark.gpu


def make_model(family):
    """-> (model, observation shape, A, EfficientZero?)"""
    import lightzero_b200 as lzb
    if family in ("atari_mz84", "atari_mz96"):
        px = int(family[-2:])
        m = lzb.MuZeroModel(observation_shape=(4, px, px), action_space_size=6, downsample=True)
        return m.load_state_dict(_conv_sd((4, px, px), 6, 5)), (4, px, px), 6, False
    m, obs, A, ez, _, _ = rezero_model(family)
    return m, obs, A, ez


FAMILIES = ["atari_mz6", "atari_mz84", "atari_mz96", "atari_ez", "connect4", "gomoku", "cartpole", "lunarlander_mz",
            "lunarlander_ez"]
_models = {}


def model_of(family):
    if family not in _models:
        _models[family] = make_model(family)
    return _models[family]


def case_inputs(case, seed, obs_shape, A):
    ctx = make_context(case, seed, A)
    T = case["N"] * case["K1"]
    g = torch.Generator().manual_seed(seed)
    obs = torch.rand((T,) + tuple(obs_shape), generator=g)
    return ctx, obs


def model_values(model, obs, mini):
    out = []
    with torch.no_grad():
        for beg in range(0, obs.shape[0], mini):
            out.append(model.initial_inference(obs[beg:beg + mini].to(model.device), return_scalar_value=True).value_scalar)
    return torch.cat(out).cpu().numpy()


def args_of(ctx):
    return (ctx["value_mask"], ctx["pos"], ctx["rewards_list"], ctx["game_segment_lens"], ctx["td_steps_list"],
            ctx["to_play_segment"])


def device_targets(model, obs, ctx, case, mini=10240, **kw):
    from lightzero_b200.reanalyze import compute_target_reward_value
    return compute_target_reward_value(model, obs, *args_of(ctx), num_unroll_steps=case["K1"] - 1,
                                       discount_factor=case["discount"], env_type=ctx["env_type"],
                                       efficientzero=case["kind"] == "ez", lstm_horizon_len=case.get("H", 5),
                                       mini_infer_size=mini, return_values=True, **kw)


def expected(values, ctx, case):
    return reward_value_targets(values, *args_of(ctx), num_unroll_steps=case["K1"] - 1, discount_factor=case["discount"],
                                env_type=ctx["env_type"], efficientzero=case["kind"] == "ez", lstm_horizon_len=case.get("H", 5))


def assert_bits(got, exp):
    for a, b, what in ((got[0], exp[0], "rewards / value prefixes"), (got[1], exp[1], "value targets")):
        assert a.dtype == np.float64 and a.shape == b.shape, what
        assert np.array_equal(a.view(np.uint64), b.view(np.uint64)), f"{what} differ"


def check(family, name, mini=10240, case=None):
    model, obs_shape, A, ez = model_of(family)
    case = case or CASES[name]
    ctx, obs = case_inputs(case, seed_of(name), obs_shape, A)
    got = device_targets(model, obs, ctx, case, mini)
    values = model_values(model, obs, mini)
    assert np.array_equal(got[2].cpu().numpy().view(np.uint32), values.view(np.uint32)), "value scalars differ"
    assert_bits(got, expected(values, ctx, case))
    return got


# every model family on a MuZero / EfficientZero case of its kind, with two mini_infer_size slicings
@pytest.mark.parametrize("family", FAMILIES)
@pytest.mark.parametrize("mini", [10240, 16])
def test_every_family(family, mini):
    ez = family.endswith("_ez")
    check(family, "ez_2p_f32_n64_k6_h5" if ez else "mz_2p_f32_n64_k6", mini)
    check(family, "ez_f32x1_n7_k6_h5" if ez else "mz_f64_n7_k6", mini)


# the whole case grid of the fixtures (use_root_value cases bootstrap from the network here; test_ez_root_value searches)
@pytest.mark.parametrize("name", sorted(CASES))
def test_case_grid(name):
    check("atari_ez" if CASES[name]["kind"] == "ez" else "atari_mz6", name)


@pytest.mark.parametrize("N", [256, 1024])
def test_atari_batch_sizes(N):
    """256 x 6 rows (the Atari default batch) and 1024 x 6"""
    case = dict(CASES["mz_f32_n7_k6"], N=N)
    check("atari_mz6", f"atari_{N}", mini=2048, case=case)
    check("atari_ez", f"atari_ez_{N}", case=dict(CASES["ez_2p_f32_n64_k6_h5"], N=N))


def test_value_scalars_within_the_scalar_contract():
    """The value scalars are h^-1 of the model's own value logits within 2e-4 (DESIGN.md §4.4), so the targets follow the
    reference pipeline (inverse_scalar_transform on the logits) up to that contract"""
    model, obs_shape, A, _ = model_of("atari_mz6")
    ctx, obs = case_inputs(CASES["mz_f32_n64_k6_td9"], 7, obs_shape, A)
    got = device_targets(model, obs, ctx, CASES["mz_f32_n64_k6_td9"])
    with torch.no_grad():
        logits = model.initial_inference(obs.to(model.device)).value.double()
    support = torch.arange(-300, 301, 1, dtype=torch.float64, device=logits.device)
    x = (torch.softmax(logits, dim=1) * support).sum(1)
    eps = 0.001
    ref = torch.sign(x) * (((torch.sqrt(1 + 4 * eps * (x.abs() + 1 + eps)) - 1) / (2 * eps)) ** 2 - 1)
    err = (got[2].double() - ref).abs().max().item()
    assert err <= 2e-4, err


# ---------------------------------------------------------------------------------------------- EfficientZero use_root_value
def mirror_root_values(model, obs, ctx, case, S, noise, noises, w=0.25):
    """game_buffer_efficientzero.py:216-240 on the existing mirrors: initial_inference, Roots.prepare, search, get_values"""
    import lightzero_b200 as lzb
    T = obs.shape[0]
    mcts = lzb.EfficientZeroMCTSCtree(dict(num_simulations=S, lstm_horizon_len=case["H"], root_noise_weight=w))
    with torch.no_grad():
        o = model.initial_inference(obs.to(model.device))
    legal = [np.nonzero(ctx["action_mask"][j])[0].tolist() for j in range(T)]
    roots = mcts.roots(T, legal)
    tp = ctx["to_play"].tolist()
    if noise:
        roots.prepare(w, [n[:len(l)].tolist() for n, l in zip(noises, legal)], [0.0] * T, o.policy_logits, tp)
    else:
        roots.prepare_no_noise([0.0] * T, o.policy_logits, tp)
    mcts.search(roots, model, o.latent_state, o.reward_hidden_state, tp)
    values = np.asarray(roots.get_values(), np.float32)
    roots.clear()
    return values


def device_root(model, obs, ctx, case, S, noise, noises, mini=10240, w=0.25):
    import lightzero_b200 as lzb
    mcts = lzb.EfficientZeroMCTSCtree(dict(num_simulations=S, lstm_horizon_len=case["H"], root_noise_weight=w))
    return device_targets(model, obs, ctx, case, mini, use_root_value=True, mcts=mcts, action_mask=ctx["action_mask"],
                          to_play=ctx["to_play"], reanalyze_noise=noise, noises=noises)


@pytest.mark.parametrize("family", ["atari_ez", "lunarlander_ez"])
@pytest.mark.parametrize("name", ["ez_root_f32_n7_k6_h5", "ez_root_2p_f32_n7_k6_h5", "ez_2p_f32_n64_k6_h5"])
@pytest.mark.parametrize("noise", [True, False])
def test_ez_root_value(family, name, noise):
    model, obs_shape, A, _ = model_of(family)
    case = CASES[name]
    ctx, obs = case_inputs(case, seed_of(name), obs_shape, A)     # masked roots: make_context draws legal-action masks
    assert (ctx["action_mask"] == 0).any()
    S = 12
    noises = ctx["noises"]
    got = device_root(model, obs, ctx, case, S, noise, noises, mini=100)
    values = mirror_root_values(model, obs, ctx, case, S, noise, noises)
    assert np.array_equal(got[2].cpu().numpy().view(np.uint32), values.view(np.uint32)), "root values differ"
    assert_bits(got, expected(values, ctx, case))


def test_repeated_root_call_captures_no_graph():
    from lightzero_b200 import cabi
    lib = cabi.load()
    model, obs_shape, A, _ = model_of("atari_ez")
    case = CASES["ez_root_f32_n7_k6_h5"]
    ctx, obs = case_inputs(case, 3, obs_shape, A)
    first = device_root(model, obs, ctx, case, 10, True, ctx["noises"])
    n0 = lib.lz_debug_graph_captures()
    second = device_root(model, obs, ctx, case, 10, True, ctx["noises"])
    assert lib.lz_debug_graph_captures() == n0, "the second call of the same shapes captured a graph"
    assert_bits(second, first)


def test_device_outputs_and_side_stream():
    """device=True returns CUDA tensors; a call on a side stream next to a busy legacy default stream gives the same bits"""
    model, obs_shape, A, _ = model_of("atari_mz6")
    case = CASES["mz_2p_f32_n64_k6"]
    ctx, obs = case_inputs(case, 11, obs_shape, A)
    ref = device_targets(model, obs, ctx, case)
    rez = CASES["ez_root_2p_f32_n7_k6_h5"]
    ezm, ez_shape, ezA, _ = model_of("atari_ez")
    ectx, eobs = case_inputs(rez, 12, ez_shape, ezA)
    eref = device_root(ezm, eobs, ectx, rez, 10, True, ectx["noises"])
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    torch.cuda._sleep(200_000_000)                  # the legacy default stream stays busy while the calls run
    with torch.cuda.stream(side):
        got = device_targets(model, obs, ctx, case, device=True)
        egot = device_root(ezm, eobs, ectx, rez, 10, True, ectx["noises"])
    torch.cuda.synchronize()
    assert got[0].is_cuda and got[0].dtype == torch.float64 and got[1].is_cuda
    assert_bits((got[0].cpu().numpy(), got[1].cpu().numpy()), ref)
    assert_bits(egot, eref)


def test_wrong_model_and_tree_pairs_raise():
    import lightzero_b200 as lzb
    from lightzero_b200.reanalyze import compute_target_reward_value
    mz, mz_shape, A, _ = model_of("cartpole")
    ezm, ez_shape, ezA, _ = model_of("lunarlander_ez")
    case = CASES["mz_f32_n7_k6"]
    ctx, obs = case_inputs(case, 1, mz_shape, A)
    base = dict(num_unroll_steps=5)
    with pytest.raises(TypeError):                   # a MuZero model with the EfficientZero buffer's call
        compute_target_reward_value(mz, obs, *args_of(ctx), efficientzero=True, **base)
    ctx2, obs2 = case_inputs(case, 1, ez_shape, ezA)
    with pytest.raises(TypeError):                   # an EfficientZero model with the MuZero buffer's call
        compute_target_reward_value(ezm, obs2, *args_of(ctx2), **base)
    for mcts in (lzb.MuZeroMCTSCtree(dict(num_simulations=4)), lzb.GumbelMuZeroMCTSCtree(dict(num_simulations=4)), None):
        with pytest.raises(TypeError):               # the root-value search needs an EfficientZeroMCTSCtree
            compute_target_reward_value(ezm, obs2, *args_of(ctx2), efficientzero=True, use_root_value=True, mcts=mcts,
                                        action_mask=ctx2["action_mask"], to_play=ctx2["to_play"], **base)
