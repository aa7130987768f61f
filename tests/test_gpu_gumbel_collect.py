"""Gumbel MuZero collect on the device (GumbelMuZeroCollectPolicy, lz_search_collect* on Gumbel trees,
lz_tree_gumbel_select_action, the segments' improved-policy array):
- forward_collect / forward_eval against GumbelMuZeroPolicy._forward_collect / _forward_eval restated on the compiled reference
  tree (oracle/build_gmz_ref.py) driving the same CUDA network: visit counts, root values, improved policies, masked completed
  values and actions bit for bit, the entropy to select_action's tolerance;
- the collect equals the step-wise GumbelMuZeroMCTSCtree.search + lz_tree_gumbel_policies on the same inputs, in one graph
  launch with no host synchronisation, re-captured after a weight reload or set_math;
- SegmentStats' improved policies against GameSegment.store_search_stats(..., improved_policy=...) restated;
- refusals.
"""
import ctypes

import numpy as np
import pytest
import torch

import board_model_ref as BR
import mlp_mz_model_ref as MR
from oracle.tree_drive import drive, network, readout
from test_gpu_search_oracle import _inputs, zero_policy

pytestmark = pytest.mark.gpu

DISCOUNT = 0.997


def _oracle():
    from oracle import build_gmz_ref
    mod = build_gmz_ref.load()
    if mod is None:
        pytest.skip("compiled reference Gumbel tree not built (oracle/build_gmz_ref.py)")
    return mod


def _model(name, seed, mutate=None):
    """(CUDA model, observation shape) of a shipped Gumbel config: Atari 64x64 conv with A = 6 / 18, tictactoe, gomoku 6x6,
    cartpole, lunarlander"""
    import lightzero_b200 as lzb
    from oracle import model_ref as R
    if name.startswith("atari"):
        A, obs = int(name[5:]), (4, 64, 64)
        ref = R.emulate_trained_(R.MuZeroModelRef(obs, A), seed)
        if mutate is not None:
            mutate(ref)
        return lzb.MuZeroModel(observation_shape=obs, action_space_size=A, downsample=True).load_state_dict(ref.state_dict()), obs
    if name in BR.BOARD_CONFIGS:
        cu = lzb.MuZeroModel(**BR.model_kwargs(name)).load_state_dict(BR.build(name, seed).state_dict())
        return cu, tuple(BR.BOARD_CONFIGS[name][0])
    if name == "cartpole":
        ref = R.emulate_trained_mlp_(R.MuZeroModelMLPRef(4, 2, res_connection_in_dynamics=True), seed)
        return lzb.MuZeroModelMLP(observation_shape=4, action_space_size=2, res_connection_in_dynamics=True).load_state_dict(
            ref.state_dict()), (4,)
    return lzb.MuZeroModelMLP(**MR.model_kwargs(name)).load_state_dict(MR.build(name, seed).state_dict()), (MR.CONFIGS[name][0],)


def _obs(shape, B, seed, u8=False):
    g = torch.Generator().manual_seed(seed)
    if u8:
        x = torch.randint(0, 256, (B,) + shape, dtype=torch.uint8, generator=g)
        return x, (x.double() / 255.0).float()        # the reference's ScaledFloatFrameWrapper
    x = torch.rand((B,) + shape, generator=g)
    return x, x


def _mask(legal, A):
    mask = np.zeros((len(legal), A), np.uint8)
    for b, l in enumerate(legal):
        mask[b, l] = 1
    return mask


def _expected(gref, cu, x, mask, legal, noises, tp, S, m, temperature):
    """GumbelMuZeroPolicy._forward_collect / _forward_eval (lzero/policy/gumbel_muzero.py:549-605, 660-707) with the compiled
    reference tree and the CUDA network's initial / recurrent inference"""
    from lightzero_b200.collect import select_action
    B, A = mask.shape
    out = cu.initial_inference(x.cuda(), return_scalar_value=True)
    c = dict(B=B, A=A, S=S, m=m, legal=legal, to_play=tp, root_logits=out.policy_logits.cpu().numpy(),
             root_values=out.value_scalar.cpu().numpy(), discount=DISCOUNT)
    if noises is not None:
        c["noises"] = noises
    t, _ = drive(gref, c, "gumbel", network(cu, out.latent_state))
    exp = []
    for i in range(B):
        dist = [int(v) for v in t["distributions"][i] if v >= 0]
        improved = t["policies"][i]
        exp.append(dict(visit_count_distributions=dist, searched_value=t["root_values_bits"][i],
                        improved_policy_probs=improved, roots_completed_value=np.where(mask[i] == 1, t["children_values"][i], 0.0),
                        action=int(np.argmax(np.where(mask[i] == 1, improved, 0.0))),
                        entropy=select_action(dist, temperature=temperature, deterministic=True)[1],
                        predicted_value=float(out.value_scalar[i])))
    return exp


def _check(got, exp, collect):
    assert len(got) == len(exp)
    keys = {'action', 'visit_count_distributions', 'visit_count_distribution_entropy', 'searched_value', 'predicted_value',
            'predicted_policy_logits'}
    if collect:
        keys |= {'roots_completed_value', 'improved_policy_probs'}
    for i, e in enumerate(exp):
        g = got[i]
        assert set(g) == keys
        assert g['visit_count_distributions'] == e['visit_count_distributions'], i
        assert np.float32(g['searched_value']).view(np.uint32) == e['searched_value'], i
        assert g['action'] == e['action'], i
        assert abs(g['visit_count_distribution_entropy'] - e['entropy']) <= 1e-6 * max(1.0, abs(e['entropy'])), i
        assert g['predicted_value'] == e['predicted_value'], i
        if collect:
            assert np.array_equal(g['improved_policy_probs'].astype(np.float32).view(np.uint32),
                                  np.asarray(e['improved_policy_probs'], np.float32).view(np.uint32)), i
            assert np.array_equal(g['roots_completed_value'].astype(np.float32).view(np.uint32),
                                  e['roots_completed_value'].astype(np.float32).view(np.uint32)), i


CASES = [  # model, B, S, m, observation path (device / host, float / uint8), players, collect (else eval)
    ("atari6", 8, 16, 4, "device", "1p", True),
    ("atari6", 8, 16, 6, "host_u8", "1p", False),
    ("atari18", 256, 16, 18, "host", "1p", True),
    ("atari18", 1, 16, 4, "device_u8", "1p", True),
    ("atari18", 8, 16, 8, "host", "1p", False),
    ("tictactoe", 8, 16, 4, "device", "2p", True),
    ("tictactoe", 256, 16, 9, "host", "2p", False),
    ("gomoku", 8, 16, 8, "host", "2p", True),
    ("cartpole", 256, 16, 2, "device", "1p", True),
    ("lunarlander", 8, 16, 4, "host", "1p", True),
    ("lunarlander", 1, 16, 2, "device", "1p", False),
]


@pytest.mark.parametrize("name,B,S,m,path,players,collect", CASES)
def test_collect_and_eval_match_reference_pipeline(name, B, S, m, path, players, collect):
    import lightzero_b200 as lzb
    gref = _oracle()
    cu, shape = _model(name, 3)
    A = cu.action_space_size
    xin, x = _obs(shape, B, 7, u8=path.endswith("u8"))
    legal, _, _, tp = _inputs(B, A, 11, players)       # masked roots, one with a single legal action
    mask = _mask(legal, A)
    pol = lzb.GumbelMuZeroCollectPolicy(cu, dict(num_simulations=S, max_num_considered_actions=m, discount_factor=DISCOUNT))
    obs = xin.pin_memory() if path.startswith("host") else xin.cuda()
    temperature = 0.5 if collect else 1.0
    np.random.seed(5)
    if collect:
        got = pol.forward_collect(obs, mask, temperature=temperature, to_play=tp)
    else:
        got = pol.forward_eval(obs, mask, to_play=tp)
    noises = None
    if collect:         # forward_collect's Dirichlet draws, in the same order
        np.random.seed(5)
        noises = [np.random.dirichlet([0.3] * len(l)).astype(np.float32).tolist() for l in legal]
    _check(got, _expected(gref, cu, x, mask, legal, noises, tp, S, m, temperature), collect)


def test_first_maximum_of_tied_improved_policy():
    """uniform priors and two simulations leave most legal actions unvisited with the same completed Q: their improved
    probabilities tie exactly and the action is the first of them, as np.argmax picks"""
    import lightzero_b200 as lzb
    gref = _oracle()
    B, S, m = 64, 2, 4
    cu, shape = _model("atari18", 4, mutate=zero_policy)
    A = cu.action_space_size
    _, x = _obs(shape, B, 9)
    legal, _, _, tp = _inputs(B, A, 12, "1p")
    mask = _mask(legal, A)
    pol = lzb.GumbelMuZeroCollectPolicy(cu, dict(num_simulations=S, max_num_considered_actions=m, discount_factor=DISCOUNT))
    got = pol.forward_eval(x.cuda(), mask, to_play=tp)
    exp = _expected(gref, cu, x, mask, legal, None, tp, S, m, 1.0)
    _check(got, exp, False)
    ties = 0
    for i, e in enumerate(exp):
        p = np.where(mask[i] == 1, e['improved_policy_probs'], 0.0)
        ties += int((p == p.max()).sum() > 1)
    assert ties > 0


def _stepwise(cu, x, legal, noises, tp, S, m):
    """GumbelMuZeroMCTSCtree.search driven step by step around the model, then lz_tree_gumbel_policies"""
    import lightzero_b200 as lzb

    class Wrapped:          # any non-lightzero_b200 model object goes through the step-wise drive
        def recurrent_inference(self, lat, act):
            return cu.recurrent_inference(lat, act)
    B, A = len(legal), cu.action_space_size
    out = cu.initial_inference(x, return_scalar_value=True)
    mcts = lzb.GumbelMuZeroMCTSCtree(dict(num_simulations=S, max_num_considered_actions=m, discount_factor=DISCOUNT))
    roots = mcts.roots(B, legal)
    roots.prepare(0.25, noises, [0.0] * B, out.value_scalar, out.policy_logits, tp)
    mcts.search(roots, Wrapped(), out.latent_state, tp)
    r = readout(roots, A, S, DISCOUNT)
    roots.clear()
    return r


def _fused_kernels(cu, x, legal, tp, S, m):
    import lightzero_b200 as lzb
    B = len(legal)
    out = cu.initial_inference(x, return_scalar_value=True)
    mcts = lzb.GumbelMuZeroMCTSCtree(dict(num_simulations=S, max_num_considered_actions=m, discount_factor=DISCOUNT))
    roots = mcts.roots(B, legal)
    roots.prepare_no_noise([0.0] * B, out.value_scalar, out.policy_logits, tp)
    mcts.search(roots, cu, out.latent_state, tp)
    roots.clear()
    return mcts.last_num_kernels


def _same_as_stepwise(got, exp, mask):
    assert np.array_equal(got["visits"].cpu().numpy(), exp["distributions"])
    assert np.array_equal(got["values"].cpu().numpy().view(np.uint32), exp["root_values_bits"])
    assert np.array_equal(got["improved_policy"].cpu().numpy().view(np.uint32), exp["policies"].view(np.uint32))
    cv = np.where(mask == 1, exp["children_values"], 0.0).astype(np.float32)
    assert np.array_equal(got["completed_values"].cpu().numpy().view(np.uint32), cv.view(np.uint32))


def test_collect_equals_stepwise_search_in_one_graph_without_host_sync():
    import lightzero_b200 as lzb
    from oracle.model_ref import MuZeroModelRef, emulate_trained_
    B, S, m = 32, 12, 4
    cu, shape = _model("atari18", 5)
    A = cu.action_space_size
    _, x = _obs(shape, B, 3)
    x = x.cuda()
    legal, _, noises, tp = _inputs(B, A, 13, "1p")
    mask = _mask(legal, A)
    noise_rows = np.zeros((B, A), np.float32)
    for b, n in enumerate(noises):
        noise_rows[b, :len(n)] = n
    d_mask, d_noise = torch.from_numpy(mask).cuda(), torch.from_numpy(noise_rows).cuda()
    d_tp = torch.tensor(tp, dtype=torch.int32).cuda()
    pol = lzb.GumbelMuZeroCollectPolicy(cu, dict(num_simulations=S, max_num_considered_actions=m, discount_factor=DISCOUNT))

    def collect():
        return pol.search_batch(x, d_mask, d_noise, d_tp, read_back=False, select=(1.0, True, 0))
    got = collect()
    _same_as_stepwise(got, _stepwise(cu, x, legal, noises, tp, S, m), mask)
    assert pol.last_num_kernels == _fused_kernels(cu, x, legal, tp, S, m) >= 1 + 2 * S
    # no host synchronisation inside a collect: the call returns while a long kernel queued before it still runs
    collect()
    torch.cuda.synchronize()
    torch.cuda._sleep(500_000_000)
    collect()
    done = torch.cuda.Event()
    done.record()
    assert not done.query()
    torch.cuda.synchronize()
    # a weight reload and then set_math re-capture the graph: the results follow the new weights / math mode
    cu.load_state_dict(emulate_trained_(MuZeroModelRef(shape, A), 9).state_dict())
    _same_as_stepwise(collect(), _stepwise(cu, x, legal, noises, tp, S, m), mask)
    cu.set_math("tc1")
    _same_as_stepwise(collect(), _stepwise(cu, x, legal, noises, tp, S, m), mask)
    cu.set_math("tc3")
    # a MuZero collect on the same pooled tree turns it back into a MuZero tree
    mz = lzb.collect.MuZeroCollectPolicy(cu, dict(num_simulations=S, deterministic=True, discount_factor=DISCOUNT))
    r = mz.search_batch(x, d_mask, d_noise, d_tp, read_back=False)
    assert (r["visits"].sum(1) + (r["visits"] < 0).sum(1) == S).all()


def test_gumbel_policies_and_select_action_agree():
    """lz_tree_gumbel_policies and lz_tree_gumbel_select_action are one read-out: the improved policy is the same bits and
    the completed values differ only in the fill at illegal actions (-inf / 0)"""
    import lightzero_b200 as lzb
    from lightzero_b200 import cabi
    B, S, m = 16, 8, 4
    cu, shape = _model("lunarlander", 2)
    A = cu.action_space_size
    _, x = _obs(shape, B, 4)
    legal, _, noises, tp = _inputs(B, A, 14, "1p")
    out = cu.initial_inference(x.cuda(), return_scalar_value=True)
    mcts = lzb.GumbelMuZeroMCTSCtree(dict(num_simulations=S, max_num_considered_actions=m))
    roots = mcts.roots(B, legal)
    roots.prepare(0.25, noises, [0.0] * B, out.value_scalar, out.policy_logits, tp)
    mcts.search(roots, cu, out.latent_state, tp)
    cv, ip = roots.get_children_values_tensor(DISCOUNT, A), roots.get_policies_tensor(DISCOUNT, A)
    t = roots._tree
    f = [torch.empty(B, A, device="cuda") for _ in range(2)]
    act, ent = torch.empty(B, dtype=torch.int32, device="cuda"), torch.empty(B, device="cuda")
    cabi.check(t.lib.lz_tree_gumbel_select_action(t.h, 1.0, act.data_ptr(), ent.data_ptr(), f[0].data_ptr(), f[1].data_ptr(),
                                                  cabi.stream_ptr()), "lz_tree_gumbel_select_action")
    _, _, ent_ref = roots.select_action_tensor(1.0, deterministic=True)
    assert torch.equal(f[1].view(torch.int32), ip.view(torch.int32))
    assert torch.equal(f[0].view(torch.int32), torch.where(torch.isinf(cv), 0.0, cv).view(torch.int32))
    assert torch.equal(ent.view(torch.int32), ent_ref.view(torch.int32))    # lz_tree_select_action's arithmetic
    for o in (None, ent):           # every output may be NULL
        cabi.check(t.lib.lz_tree_gumbel_select_action(t.h, 1.0, act.data_ptr(), cabi.ptr(o), None, None, cabi.stream_ptr()), "NULL")
    assert t.lib.lz_tree_gumbel_select_action(t.h, 0.0, None, None, None, None, cabi.stream_ptr()) == -1
    roots.clear()


def test_segment_improved_policies_follow_store_search_stats():
    """k collect steps with a mix of active environments, a reset of some, and segments that fill up: the improved-policy
    array holds what GameSegment.store_search_stats(..., improved_policy=...) appends per environment, zero elsewhere"""
    import lightzero_b200 as lzb
    from lightzero_b200.collector import SegmentStats
    B, T, S, m = 8, 4, 8, 4
    cu, shape = _model("tictactoe", 6)
    A = cu.action_space_size
    rng = np.random.default_rng(3)
    pol = lzb.GumbelMuZeroCollectPolicy(cu, dict(num_simulations=S, max_num_considered_actions=m))
    seg = SegmentStats(B, T, A)
    assert seg.improved_policy() is None
    lists = [[] for _ in range(B)]
    for step in range(7):
        if step == 3:
            done = rng.random(B) < 0.5
            seg.reset(torch.from_numpy(done.astype(np.uint8)))
            for b in np.nonzero(done)[0]:
                lists[b] = []
        _, x = _obs(shape, B, 100 + step)
        legal, _, noises, tp = _inputs(B, A, 200 + step, "2p")
        r = pol.search_batch(x.cuda(), torch.from_numpy(_mask(legal, A)).cuda(), None, tp, read_back=False, select=(1.0, True, 0))
        active = rng.random(B) < 0.7
        seg.store_search_stats(r["visits"], r["values"], torch.from_numpy(active.astype(np.uint8)), improved_policy=r["improved_policy"])
        ip = r["improved_policy"].cpu().numpy()
        for b in np.nonzero(active)[0]:
            if len(lists[b]) < T:            # a full segment is left unchanged
                lists[b].append(ip[b])
    exp = np.zeros((B, T, A), np.float32)
    for b, l in enumerate(lists):
        if l:
            exp[b, :len(l)] = np.stack(l)
    _, _, lens = seg.tensors()
    assert lens.cpu().tolist() == [len(l) for l in lists]
    assert np.array_equal(seg.improved_policy().cpu().numpy().view(np.uint32), exp.view(np.uint32))
    seg.reset()
    assert not seg.improved_policy().any() and not seg.tensors()[2].any()


def test_refusals():
    import lightzero_b200 as lzb
    from lightzero_b200 import cabi, mz_tree
    with pytest.raises(TypeError):
        lzb.GumbelMuZeroCollectPolicy(lzb.EfficientZeroModel.__new__(lzb.EfficientZeroModel))
    with pytest.raises(TypeError):
        lzb.GumbelMuZeroCollectPolicy(lzb.EfficientZeroModelMLP.__new__(lzb.EfficientZeroModelMLP))
    # a search of more simulations than the tree's Gumbel num_simulations: LZ_EINVAL with a message, before any work
    cu, shape = _model("cartpole", 1)
    B, A = 4, 2
    tree = mz_tree.acquire_tree(torch.device("cuda", torch.cuda.current_device()), B, A, 8)
    try:
        lib = tree.lib
        cabi.check(lib.lz_tree_set_gumbel(tree.h, A, 4), "lz_tree_set_gumbel")
        q = tree.search_for(cu, 8, ("gumbel",))
        obs = torch.rand((B,) + shape, device="cuda")
        rc = lib.lz_search_collect(q, obs.data_ptr(), None, None, 0.0, None, 1, None, None, cabi.stream_ptr())
        assert rc == -1 and b"considered-visit table" in lib.lz_last_error()
        h_obs = obs.cpu().pin_memory()
        rc = lib.lz_search_collect_host(q, h_obs.data_ptr(), None, None, 0.0, None, 1, 1, None, None, cabi.stream_ptr())
        assert rc == -1 and b"considered-visit table" in lib.lz_last_error()
        cabi.check(lib.lz_tree_set_gumbel(tree.h, 0, 0), "lz_tree_set_gumbel off")
    finally:
        tree.release()
    # uint8 frames stay the conv model's: board and MLP models refuse them on Gumbel trees too
    for name in ("tictactoe", "cartpole"):
        cu, shape = _model(name, 1)
        A = cu.action_space_size
        pol = lzb.GumbelMuZeroCollectPolicy(cu, dict(num_simulations=4, max_num_considered_actions=A))
        u8 = torch.zeros((2,) + shape, dtype=torch.uint8)
        for o in (u8.cuda(), u8.pin_memory()):
            with pytest.raises(cabi.LzError, match="uint8"):
                pol.search_batch(o, np.ones((2, A), np.uint8), None, None, select=(1.0, True, 0))
    torch.cuda.synchronize()
