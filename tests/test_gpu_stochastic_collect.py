"""Stochastic MuZero collect on the device (StochasticMuZeroCollectPolicy, lz_search_collect* on stochastic trees):
- search_batch equals the step-wise pipeline on the same inputs -- initial_inference, stochastic_mz_tree.Roots.prepare and
  StochasticMuZeroMCTSCtree.search -- bit for bit with the chance draw pinned (chance_seed): visits, root-value bits, the
  predicted value and the first A logit columns, for the three shipped configs (C > A, A > C, A >> C), device and pinned-host
  observations (1 and 3 copy chunks), masked and unmasked roots, one and two players, collect and eval, B up to 1024.  The
  step-wise search equals the compiled reference tree driving the same network (tests/test_gpu_stochastic.py::test_tree_parity);
- forward_collect / forward_eval return the reference's output dicts; device select_action reads only the legal children,
  repeats for a fixed seed and samples the visit distribution;
- sampled chance draws (chance_seed=None): successive steps draw afresh, at the afterstate policy's frequencies, and a step on a
  fresh tree repeats the step-wise search on another fresh tree with the same RNG key bit for bit;
- SegmentStats stores the first A of the tree's W visit columns;
- compute_target_reward_value with a StochasticMuZeroModelMLP gives the MuZero buffer's targets;
- the collect on a side stream next to a busy legacy default stream (tests/test_gpu_streams.py's harness);
- one captured graph of 3S + 1 kernels per shape.
"""
import numpy as np
import pytest
import torch

import stoch_mlp_model_ref as SR
from test_gpu_streams import _check_on_side_stream, sleep_rate  # noqa: F401  (the streams harness and its fixture)

pytestmark = pytest.mark.gpu

DISCOUNT = 0.997
_models = {}


def model(name):
    """The CUDA StochasticMuZeroModelMLP of a config, with the reference class's weights (one per config for the module)"""
    import lightzero_b200 as lzb
    if name not in _models:
        sd = SR.build(name, list(SR.CONFIGS).index(name)).state_dict()
        _models[name] = lzb.StochasticMuZeroModelMLP(**SR.model_kwargs(name)).load_state_dict(sd)
    return _models[name]


def inputs(name, B, masked, two_player, seed):
    """(obs [B, obs_dim] f32 host, mask uint8 [B, A], noises f32 [B, A] in legal order, to_play int32 [B])"""
    obs_dim, A = SR.CONFIGS[name][:2]
    rng = np.random.default_rng(seed)
    obs = rng.uniform(-1, 1, (B, obs_dim)).astype(np.float32)
    mask = np.ones((B, A), np.uint8)
    if masked:
        mask = (rng.random((B, A)) < 0.6).astype(np.uint8)
        mask[np.arange(B), rng.integers(0, A, B)] = 1
        mask[0] = 0
        mask[0, A - 1] = 1                  # a root with its last action as the only legal one
    noises = np.zeros((B, A), np.float32)
    for b in range(B):
        n = int(mask[b].sum())
        noises[b, :n] = rng.dirichlet([0.3] * n)
    to_play = rng.integers(1, 3, B).astype(np.int32) if two_player else np.full(B, -1, np.int32)
    return obs, mask, noises, to_play


def stepwise(cu, obs, mask, noises, to_play, S, chance_seed, keep=False):
    """The reference-shaped pipeline: initial_inference, Roots.prepare (prepare_no_noise when noises is None) and
    StochasticMuZeroMCTSCtree.search on the same network; returns the device read-out (and the roots when keep)"""
    import lightzero_b200 as lzb
    B = obs.shape[0]
    o = cu.initial_inference(torch.from_numpy(obs).cuda(), return_scalar_value=True)
    mcts = lzb.StochasticMuZeroMCTSCtree(dict(num_simulations=S, deterministic=True, chance_seed=chance_seed,
                                              discount_factor=DISCOUNT))
    roots = mcts.roots(B, mask, cu.chance_space_size)
    if noises is None:
        roots.prepare_no_noise([0.] * B, o.policy_logits, to_play)
    else:
        roots.prepare(0.25, noises, [0.] * B, o.policy_logits, to_play)
    mcts.search(roots, cu, o.latent_state, to_play)
    visits, nl = roots.get_distributions_tensor()
    out = dict(visits=visits.clone(), values=roots.get_values_tensor().clone(), nlegal=nl.clone(), pred_value=o.value_scalar,
               policy_logits=o.policy_logits)
    if keep:
        return out, roots
    roots.clear()
    return out


def policy(cu, S, chance_seed, **kw):
    import lightzero_b200 as lzb
    return lzb.StochasticMuZeroCollectPolicy(cu, dict(num_simulations=S, deterministic=True, chance_seed=chance_seed,
                                                      discount_factor=DISCOUNT, **kw))


def assert_same(got, exp, A):
    for k in ("visits", "nlegal"):
        assert torch.equal(got[k].cuda(), exp[k]), k
    for k in ("values", "pred_value"):
        assert np.array_equal(got[k].cpu().numpy().view(np.uint32), exp[k].cpu().numpy().view(np.uint32)), k
    g = got["policy_logits"].cpu().numpy()
    assert g.shape == (exp["policy_logits"].shape[0], A)
    assert np.array_equal(g.view(np.uint32), exp["policy_logits"].cpu().numpy().view(np.uint32))


CASES = [  # config, B, S, observation path (device / host with 1 or 3 chunks), masked, two players, collect (else eval)
    ("cartpole", 1024, 25, "device", False, False, True),
    ("cartpole", 1024, 25, "host3", True, False, True),
    ("cartpole", 37, 25, "host1", True, True, False),
    ("lunarlander_disc", 8, 50, "device", True, False, True),
    ("lunarlander_disc", 300, 50, "host3", False, True, True),
    ("lunarlander_disc", 1024, 50, "device", True, False, False),
    ("pendulum_cont_disc", 200, 50, "host1", True, False, True),
    ("pendulum_cont_disc", 64, 50, "device", False, True, False),
]


@pytest.mark.parametrize("name,B,S,path,masked,two_player,collect", CASES)
def test_collect_equals_stepwise(name, B, S, path, masked, two_player, collect):
    cu = model(name)
    A = cu.action_space_size
    obs, mask, noises, to_play = inputs(name, B, masked, two_player, B + S)
    noises = noises if collect else None
    exp = stepwise(cu, obs, mask, noises, to_play, S, 77)
    pol = policy(cu, S, 77)
    if path == "device":
        x, m, nz = torch.from_numpy(obs).cuda(), torch.from_numpy(mask).cuda(), None if noises is None else torch.from_numpy(noises).cuda()
    else:
        pol.h2d_chunks = int(path[-1])
        x, m, nz = torch.from_numpy(obs).pin_memory(), mask, noises
    got = pol.search_batch(x, m, nz, to_play, read_back=False)
    assert got["visits"].shape == (B, max(A, cu.chance_space_size))
    assert_same(got, exp, A)
    v = got["visits"]
    assert bool((torch.where(v > 0, v, 0).sum(1) == S).all())
    assert torch.equal((got["visits"] >= 0).sum(1), got["nlegal"])
    # the read-back path gives the same numbers in pinned host tensors
    host = pol.search_batch(x, m, nz, to_play)
    assert_same(host, exp, A)


def test_forward_dicts():
    """forward_collect / forward_eval: the reference's keys and lengths; eval's action is the first maximum of the visits;
    one stream synchronisation per call at B = 1024"""
    name, B, S = "cartpole", 1024, 25
    cu = model(name)
    A = cu.action_space_size
    obs, mask, _, to_play = inputs(name, B, True, False, 5)
    pol = policy(cu, S, 3)
    x = torch.from_numpy(obs).pin_memory()
    syncs = []
    sync = torch.cuda.Stream.synchronize
    torch.cuda.Stream.synchronize = lambda self: (syncs.append(1), sync(self))[1]
    np.random.seed(0)           # the root noise
    try:
        out = pol.forward_collect(x, mask, temperature=1.0, to_play=to_play)
    finally:
        torch.cuda.Stream.synchronize = sync
    assert len(syncs) == 1
    ev = pol.forward_eval(x, mask, to_play=to_play)
    keys = {'action', 'visit_count_distributions', 'visit_count_distribution_entropy', 'searched_value', 'predicted_value',
            'predicted_policy_logits'}
    for o in (out, ev):
        assert sorted(o) == list(range(B))
        for i in range(B):
            legal = np.nonzero(mask[i])[0]
            assert set(o[i]) == keys
            assert len(o[i]['visit_count_distributions']) == len(legal)
            assert len(o[i]['predicted_policy_logits']) == A
            assert o[i]['action'] in legal
    for i in range(B):
        legal = np.nonzero(mask[i])[0]
        assert ev[i]['action'] == legal[int(np.argmax(ev[i]['visit_count_distributions']))]
    # device select_action: the same actions for the same seed; arg-max equals the host's choice
    np.random.seed(0)
    d1 = pol.forward_collect(x, mask, 1.0, to_play, device_select_action=True, seed=9)
    np.random.seed(0)
    d2 = pol.forward_collect(x, mask, 1.0, to_play, device_select_action=True, seed=9)
    assert [d1[i]['action'] for i in range(B)] == [d2[i]['action'] for i in range(B)]
    for i in range(B):
        assert d1[i]['action'] in np.nonzero(mask[i])[0]
        assert d1[i]['visit_count_distributions'] == out[i]['visit_count_distributions']
        assert abs(d1[i]['visit_count_distribution_entropy'] - out[i]['visit_count_distribution_entropy']) <= 1e-6


@pytest.mark.parametrize("name", ["cartpole", "lunarlander_disc"])
def test_device_select_action_frequencies(name):
    """temperature 1 over 2^13 identical roots (the search repeats exactly with the chance draw pinned): the device-chosen
    actions follow the visit distribution within 5 sigma, and are legal action ids < A"""
    cu = model(name)
    A, C = cu.action_space_size, cu.chance_space_size
    B, S = 1 << 13, 16
    obs = np.repeat(inputs(name, 1, False, False, 3)[0], B, 0)
    mask = np.ones((B, A), np.uint8)
    mask[:, 0] = 0                          # legal ids start at 1: positions and ids differ
    pol = policy(cu, S, 21)
    r = pol.search_batch(torch.from_numpy(obs).cuda(), torch.from_numpy(mask).cuda(), None, None, read_back=False,
                         select=(1.0, False, 1234))
    visits = r["visits"].cpu().numpy()
    assert (visits == visits[0]).all() and visits.shape == (B, max(A, C))
    n = A - 1
    p = visits[0, :n] / visits[0, :n].sum()
    act = r["action"].cpu().numpy()
    assert act.min() >= 1 and act.max() < A
    counts = np.bincount(act - 1, minlength=n)[:n]
    sigma = np.sqrt(B * p * (1 - p))
    assert np.all(np.abs(counts - B * p) <= 5 * sigma + 1), (counts, B * p)


def _pooled_trajectories(B, W, S):
    """get_trajectories of the pooled tree the last collect of this shape used (the only one of its shape)"""
    from lightzero_b200 import cabi, mz_tree
    t = mz_tree.acquire_tree(torch.device("cuda", torch.cuda.current_device()), B, W, S)
    try:
        cabi.check(t.lib.lz_tree_results(t.h, None, None, None, t.traj.data_ptr(), cabi.stream_ptr()), "lz_tree_results")
        return t.traj.cpu().numpy()
    finally:
        t.release()


def test_sampled_chance_draws_differ_between_steps():
    """chance_seed=None, one legal action per root, S = 2: the second descent of every tree draws the outcome of the chance
    node under the root's action.  Two steps on identical inputs draw afresh (the collect's reset advances the RNG epoch):
    each step's outcomes follow the afterstate policy within 5 sigma, and the two agree only as often as independent
    draws do"""
    name, B, S = "cartpole", 1 << 14, 2
    cu = model(name)
    A, C = cu.action_space_size, cu.chance_space_size
    obs = np.repeat(inputs(name, 1, False, False, 4)[0], B, 0)
    mask = np.zeros((B, A), np.uint8)
    mask[:, 1] = 1
    pol = policy(cu, S, None)
    x, m = torch.from_numpy(obs).cuda(), torch.from_numpy(mask).cuda()
    draws = []
    for _ in range(2):
        pol.search_batch(x, m, None, None)
        tr = _pooled_trajectories(B, max(A, C), S)
        assert (tr[:, 0] == 1).all()
        draws.append(tr[:, 1])
    lat = cu.initial_inference(x[:1]).latent_state
    after = cu.recurrent_inference(lat, torch.ones(1, dtype=torch.int32).cuda(), afterstate=False)
    p = torch.softmax(after.policy_logits[0].double(), -1).cpu().numpy()
    for d in draws:
        counts = np.bincount(d, minlength=C)
        assert len(counts) == C
        sigma = np.sqrt(B * p * (1 - p))
        assert np.all(np.abs(counts - B * p) <= 5 * sigma + 1), (counts, B * p)
    q = float((p * p).sum())
    same = int((draws[0] == draws[1]).sum())
    assert abs(same - B * q) <= 5 * np.sqrt(B * q * (1 - q)) + 1, (same, B * q)


def test_sampled_step_repeats_for_a_fixed_key():
    """chance_seed=None: the collect on a fresh tree and the step-wise search on another fresh tree have the same RNG key
    (seed, epoch 1) and the same steps, so the sampled step repeats bit for bit; a pinned chance_seed draws otherwise"""
    from lightzero_b200 import cabi
    name, B, S = "lunarlander_disc", 83, 19       # a shape no other test pools: both trees are fresh
    cu = model(name)
    A = cu.action_space_size
    obs, mask, noises, to_play = inputs(name, B, True, False, 6)
    exp, roots = stepwise(cu, obs, mask, noises, to_play, S, None, keep=True)     # holds its tree: the collect takes another
    pol = policy(cu, S, None)
    got = pol.search_batch(torch.from_numpy(obs).cuda(), mask, noises, to_play, read_back=False)
    key = []
    from lightzero_b200 import mz_tree
    t2 = mz_tree.acquire_tree(roots.device, B, max(A, cu.chance_space_size), S)
    try:
        assert t2 is not roots._tree
        for t in (roots._tree, t2):
            seed, epoch, counter = (cabi.ctypes.c_uint64(), cabi.ctypes.c_uint64(), cabi.ctypes.c_uint32())
            cabi.check(t.lib.lz_tree_debug_rng(t.h, cabi.ctypes.byref(seed), cabi.ctypes.byref(epoch), cabi.ctypes.byref(counter)),
                       "lz_tree_debug_rng")
            key.append((seed.value, epoch.value))
    finally:
        t2.release()
    roots.clear()
    assert key[0] == key[1] and key[0][1] == 1
    assert_same(got, exp, A)
    pinned = policy(cu, S, 4321).search_batch(torch.from_numpy(obs).cuda(), mask, noises, to_play, read_back=False)
    assert not torch.equal(pinned["visits"], got["visits"])


@pytest.mark.parametrize("name", ["cartpole", "lunarlander_disc"])
def test_segment_stats_store_first_a_columns(name):
    from lightzero_b200.collector import SegmentStats
    cu = model(name)
    A = cu.action_space_size
    B, S, T = 48, 25, 3
    seg = SegmentStats(B, T, A)
    pol = policy(cu, S, 8)
    want = []
    for step in range(2):
        obs, mask, noises, to_play = inputs(name, B, True, False, 40 + step)
        r = pol.search_batch(torch.from_numpy(obs).cuda(), torch.from_numpy(mask).cuda(), torch.from_numpy(noises).cuda(),
                             to_play, read_back=False)
        seg.store_search_stats(r["visits"], r["values"])
        v = r["visits"][:, :A].cpu().numpy().astype(np.int64)
        assert (r["visits"][:, A:] == -1).all()
        pos = np.where(v > 0, v, 0)
        want.append(((pos / pos.sum(1, keepdims=True)).astype(np.float32), r["values"].cpu().numpy()))
    child, values, lens = seg.tensors()
    assert child.shape == (B, T, A)
    assert (lens.cpu().numpy() == 2).all()
    for t, (c, v) in enumerate(want):
        assert np.array_equal(child[:, t].cpu().numpy(), c)
        assert np.array_equal(values[:, t].cpu().numpy(), v)


@pytest.mark.parametrize("case_name", ["mz_f32_n7_k6", "mz_f64_n64_k6_td9_d1", "mz_2p_f32_n64_k6", "mz_2p_f32_n7_k1_td1"])
def test_value_targets(case_name):
    """StochasticMuZeroGameBuffer inherits MuZeroGameBuffer._compute_target_reward_value: the device targets with the
    stochastic model equal oracle/targets_ref.py bootstrapped from that model's own initial_inference values"""
    from oracle.targets_ref import reward_value_targets
    from lightzero_b200.reanalyze import compute_target_reward_value
    from value_targets_cases import CASES as VCASES, make_context, seed_of
    case = VCASES[case_name]
    cu = model("lunarlander_disc")
    seed = seed_of(case_name)
    ctx = make_context(case, seed, cu.action_space_size)
    T = case["N"] * case["K1"]
    obs = torch.rand((T, cu.observation_shape), generator=torch.Generator().manual_seed(seed))
    args = (ctx["value_mask"], ctx["pos"], ctx["rewards_list"], ctx["game_segment_lens"], ctx["td_steps_list"],
            ctx["to_play_segment"])
    kw = dict(num_unroll_steps=case["K1"] - 1, discount_factor=case["discount"], env_type=ctx["env_type"])
    got = compute_target_reward_value(cu, obs, *args, mini_infer_size=40, return_values=True, **kw)
    values = torch.cat([cu.initial_inference(obs[b:b + 40].cuda(), return_scalar_value=True).value_scalar
                        for b in range(0, T, 40)]).cpu().numpy()
    assert np.array_equal(got[2].cpu().numpy().view(np.uint32), values.view(np.uint32))
    exp = reward_value_targets(values, *args, **kw)
    for a, b in zip(got[:2], exp[:2]):
        assert a.dtype == np.float64 and a.shape == b.shape
        assert np.array_equal(a.view(np.uint64), np.asarray(b, np.float64).view(np.uint64))


@pytest.mark.parametrize("path", ["device", "host"])
def test_collect_on_side_stream(sleep_rate, path):
    import lightzero_b200 as lzb
    name, B, S = "cartpole", 96, 25
    sd = SR.build(name, list(SR.CONFIGS).index(name)).state_dict()
    obs, mask, noises, to_play = inputs(name, B, True, True, 12)
    if path == "device":
        x, m, nz = torch.from_numpy(obs).cuda(), torch.from_numpy(mask).cuda(), torch.from_numpy(noises).cuda()
    else:
        x, m, nz = torch.from_numpy(obs).pin_memory(), torch.from_numpy(mask), torch.from_numpy(noises)

    def scenario():
        cu = lzb.StochasticMuZeroModelMLP(**SR.model_kwargs(name)).load_state_dict(sd)
        pol = policy(cu, S, 17)
        r = pol.search_batch(x, m, nz, to_play, read_back=False, select=(1.0, False, 5))
        return dict({k: v.clone() for k, v in r.items()}, _keep=(cu, pol))
    _check_on_side_stream(sleep_rate, "stochastic collect " + path, scenario)


@pytest.mark.parametrize("name,S", [("cartpole", 25), ("pendulum_cont_disc", 50)])
def test_one_graph_per_shape(name, S):
    """a repeated collect step replays the captured graph of 3S + 1 kernels: no new capture"""
    from lightzero_b200 import cabi
    cu = model(name)
    B = 128
    obs, mask, noises, to_play = inputs(name, B, True, False, 2)
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
