"""Gumbel MuZero on the device (csrc/gumbel.cu, lightzero_b200.gmz_tree, GumbelMuZeroMCTSCtree) against the compiled
reference tree ctree_gumbel_muzero (oracle/build_gmz_ref.py), bit for bit:
- the step-wise tree fed identical synthetic network outputs (quantised so that scores tie exactly and -inf fallbacks
  happen), compared per simulation (ix, iy, last action, search length, virtual to_play) and at the end (visit counts,
  root values, improved policies, completed values, trajectories);
- the fused search (one CUDA graph) against the reference tree driving the same CUDA network;
- refusals: descents past num_simulations, MuZero calls on a Gumbel tree, Gumbel runs on EfficientZero models.
"""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _oracle():
    from oracle import build_gmz_ref
    mod = build_gmz_ref.load()
    if mod is None:
        pytest.skip("compiled reference Gumbel tree not built (oracle/build_gmz_ref.py)")
    return mod


def _bits(x):
    return np.asarray(x, np.float32).view(np.uint32)


def _legal(rng, B, A, kind):
    if kind == "full":
        return [list(range(A)) for _ in range(B)]
    out = []
    for b in range(B):
        if kind == "single" or (kind == "mixed" and b % 3 == 0):
            out.append([int(rng.integers(A))])
        else:
            n = int(rng.integers(1, A + 1))
            out.append(sorted(rng.choice(A, n, replace=False).tolist()))
    return out


def _q(rng, shape, step):
    return (np.round(rng.normal(size=shape) / step) * step).astype(np.float32)


def _drive(mod, roots, B, A, S, m, legal, rng_seed, noise, to_play, discount=0.997):
    """Runs the reference search loop (mcts_ctree.py:1104-1172) with synthetic network outputs on module `mod`
    (the compiled reference or lightzero_b200.gmz_tree); returns the per-simulation records and the read-outs."""
    rng = np.random.default_rng(rng_seed)
    logits = _q(rng, (B, A), 0.5)
    values = _q(rng, (B,), 0.25)
    rewards = [0.0] * B
    tp = [to_play] * B
    if noise:
        noises = [rng.dirichlet([0.3] * len(l)).astype(np.float32).tolist() for l in legal]
        roots.prepare(0.25, noises, rewards, values.tolist(), logits.tolist(), tp)
    else:
        roots.prepare_no_noise(rewards, values.tolist(), logits.tolist(), tp)
    mm = mod.MinMaxStatsList(B)
    mm.set_delta(0.01)
    recs = []
    for sim in range(S):
        res = mod.ResultsWrapper(B)
        ix, iy, la, vtp = mod.batch_traverse(roots, S, m, discount, res, list(tp))
        recs.append((list(ix), list(iy), list(la), list(res.get_search_len()), list(vtp)))
        r = _q(rng, (B,), 0.5)
        v = _q(rng, (B,), 0.25)
        pl = _q(rng, (B, A), 1.0)
        mod.batch_back_propagate(sim + 1, discount, r.tolist(), v.tolist(), pl.tolist(), mm, res, list(vtp))
    out = dict(dist=roots.get_distributions(), values=roots.get_values(), traj=roots.get_trajectories(),
               pol=roots.get_policies(discount, A), cv=roots.get_children_values(discount, A))
    return recs, out


def _compare(exp, got):
    (erec, eout), (grec, gout) = exp, got
    for sim, (e, g) in enumerate(zip(erec, grec)):
        assert e == g, f"simulation {sim}: reference {e} != device {g}"
    assert eout["dist"] == gout["dist"]
    assert np.array_equal(_bits(eout["values"]), _bits(gout["values"]))
    assert eout["traj"] == gout["traj"]
    assert np.array_equal(_bits(eout["pol"]), _bits(gout["pol"]))
    assert np.array_equal(_bits(eout["cv"]), _bits(gout["cv"]))


CASES = [  # B, A, S, m, legal kind, noise, to_play
    (1, 1, 16, 1, "full", False, -1),
    (7, 2, 16, 2, "full", True, -1),
    (7, 6, 50, 4, "mixed", True, -1),
    (131, 6, 50, 6, "mixed", False, 1),
    (131, 18, 50, 18, "mixed", True, -1),
    (131, 18, 50, 40, "full", False, 2),
    (7, 33, 200, 33, "mixed", True, -1),
    (7, 82, 50, 82, "mixed", False, -1),
    (1024, 18, 50, 18, "mixed", True, -1),
    (16, 6, 1, 4, "mixed", True, -1),
    (16, 6, 16, 1, "single", False, -1),
]


@pytest.mark.parametrize("B,A,S,m,kind,noise,to_play", CASES)
def test_stepwise_tree_matches_reference(B, A, S, m, kind, noise, to_play):
    ref = _oracle()
    from lightzero_b200 import gmz_tree
    legal = _legal(np.random.default_rng(B * 1000 + A), B, A, kind)
    seed = B + 7 * A + S + m
    exp = _drive(ref, ref.Roots(B, legal), B, A, S, m, legal, seed, noise, to_play)
    roots = gmz_tree.Roots(B, legal)
    got = _drive(gmz_tree, roots, B, A, S, m, legal, seed, noise, to_play)
    _compare(exp, got)
    roots.clear()


def _conv_model(A, obs, seed):
    import lightzero_b200 as lzb
    from oracle.model_ref import MuZeroModelRef, emulate_trained_
    ref = emulate_trained_(MuZeroModelRef(obs, A), seed)
    return lzb.MuZeroModel(observation_shape=obs, action_space_size=A, downsample=True).load_state_dict(ref.state_dict())


def _mlp_model(A, seed):
    import lightzero_b200 as lzb
    from oracle.model_ref import MuZeroModelMLPRef, emulate_trained_mlp_
    ref = emulate_trained_mlp_(MuZeroModelMLPRef(4, A, res_connection_in_dynamics=True), seed)
    return lzb.MuZeroModelMLP(observation_shape=4, action_space_size=A, res_connection_in_dynamics=True).load_state_dict(ref.state_dict())


def _roots_inputs(model, B, A, obs, seed, masked):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand((B,) + (obs if isinstance(obs, tuple) else (obs,)), generator=g)
    out = model.initial_inference(x.cuda(), return_scalar_value=True)
    rng = np.random.default_rng(seed)
    legal = _legal(rng, B, A, "mixed" if masked else "full")
    noises = [rng.dirichlet([0.3] * len(l)).astype(np.float32).tolist() for l in legal]
    return out, legal, noises


def _oracle_search(ref, model, out, legal, noises, B, A, S, m, discount=0.997):
    """The reference tree picks every leaf, the CUDA network evaluates it (recurrent_inference(return_scalars=True))."""
    roots = ref.Roots(B, legal)
    roots.prepare(0.25, noises, [0.0] * B, out.value_scalar.cpu().tolist(), out.policy_logits.cpu().numpy().tolist(), [-1] * B)
    mm = ref.MinMaxStatsList(B)
    mm.set_delta(0.01)
    pool = [out.latent_state]
    for sim in range(S):
        res = ref.ResultsWrapper(B)
        ix, iy, la, vtp = ref.batch_traverse(roots, S, m, discount, res, [-1] * B)
        lat = torch.stack([pool[i][j] for i, j in zip(ix, iy)])
        o = model.recurrent_inference(lat, torch.tensor(la), return_scalars=True)
        pool.append(o.latent_state)
        ref.batch_back_propagate(sim + 1, discount, o.reward_scalar.cpu().tolist(), o.value_scalar.cpu().tolist(),
                                 o.policy_logits.cpu().numpy().tolist(), mm, res, vtp)
    return dict(dist=roots.get_distributions(), values=roots.get_values(), pol=roots.get_policies(discount, A),
                cv=roots.get_children_values(discount, A), traj=roots.get_trajectories())


def _fused_search(model, out, legal, noises, B, A, S, m):
    import lightzero_b200 as lzb
    mcts = lzb.GumbelMuZeroMCTSCtree(dict(num_simulations=S, max_num_considered_actions=m))
    roots = mcts.roots(B, legal)
    roots.prepare(0.25, noises, [0.0] * B, out.value_scalar, out.policy_logits, [-1] * B)
    mcts.search(roots, model, out.latent_state, [-1] * B)
    res = dict(dist=roots.get_distributions(), values=roots.get_values(), pol=roots.get_policies(0.997, A),
               cv=roots.get_children_values(0.997, A), traj=roots.get_trajectories())
    return res, mcts, roots


def _same(e, g):
    assert e["dist"] == g["dist"]
    assert np.array_equal(_bits(e["values"]), _bits(g["values"]))
    assert np.array_equal(_bits(e["pol"]), _bits(g["pol"]))
    assert np.array_equal(_bits(e["cv"]), _bits(g["cv"]))
    assert e["traj"] == g["traj"]


@pytest.mark.parametrize("obs,A,m,S,B,masked", [
    ((4, 64, 64), 18, 18, 50, 1, False),
    ((4, 64, 64), 18, 18, 50, 131, True),
    ((4, 64, 64), 18, 18, 50, 1024, False),
    ((4, 96, 96), 6, 4, 50, 131, True),
    ((4, 64, 64), 33, 8, 16, 64, True),
    (4, 2, 2, 50, 131, False),          # MuZeroModelMLP (the CartPole Gumbel config)
])
def test_fused_search_matches_reference_driving_the_same_network(obs, A, m, S, B, masked):
    ref = _oracle()
    model = _mlp_model(A, 5) if obs == 4 else _conv_model(A, obs, 3)
    out, legal, noises = _roots_inputs(model, B, A, obs, 11, masked)
    got, mcts, roots = _fused_search(model, out, legal, noises, B, A, S, m)
    assert mcts.last_num_kernels >= 1 + 2 * S
    _same(_oracle_search(ref, model, out, legal, noises, B, A, S, m), got)
    roots.clear()


def test_fused_equals_stepwise_and_recaptures():
    import lightzero_b200 as lzb
    A, B, S, m, obs = 18, 64, 16, 18, (4, 64, 64)
    model = _conv_model(A, obs, 4)
    out, legal, noises = _roots_inputs(model, B, A, obs, 2, True)
    fused, mcts, roots = _fused_search(model, out, legal, noises, B, A, S, m)

    class Wrapped:           # any non-lightzero_b200 model object goes through the step-wise drive
        def recurrent_inference(self, lat, act):
            return model.recurrent_inference(lat, act)
    roots2 = mcts.roots(B, legal)
    roots2.prepare(0.25, noises, [0.0] * B, out.value_scalar, out.policy_logits, [-1] * B)
    mcts.search(roots2, Wrapped(), out.latent_state, [-1] * B)
    _same(fused, dict(dist=roots2.get_distributions(), values=roots2.get_values(), pol=roots2.get_policies(0.997, A),
                      cv=roots2.get_children_values(0.997, A), traj=roots2.get_trajectories()))
    roots2.clear()
    # a weight reload and then a parameter change must re-capture the graph the first search captured on this pooled tree:
    # results follow the new weights / (m, S)
    tree = roots._tree
    roots.clear()
    ref = _oracle()
    from oracle.model_ref import MuZeroModelRef, emulate_trained_
    model.load_state_dict(emulate_trained_(MuZeroModelRef(obs, A), 9).state_dict())
    for mm_ in (m, 4):
        got, _, r = _fused_search(model, out, legal, noises, B, A, S, mm_)
        assert r._tree is tree            # the same tree and search handle, whose graph was captured before
        _same(_oracle_search(ref, model, out, legal, noises, B, A, S, mm_), got)
        r.clear()


def _golden():
    import glob
    import os
    import sys
    from conftest import GOLDEN_DIR
    sys.path.insert(0, GOLDEN_DIR)
    import make_gumbel_golden
    files = sorted(glob.glob(os.path.join(GOLDEN_DIR, "gumbel_*.npz")))
    assert len(files) == len(make_gumbel_golden.CASES)
    return make_gumbel_golden, files


def test_golden_fixtures_replay_on_device():
    """tests/golden/gumbel_*.npz (written from the compiled reference) replayed through lightzero_b200.gmz_tree, with no
    reference module involved: per-simulation leaf choices and virtual to_play, and the read-outs, bit for bit."""
    from lightzero_b200 import gmz_tree
    gen, files = _golden()
    for f in files:
        d = dict(np.load(f))
        got = gen.replay(gmz_tree, d)
        for k in gen.EXPECTED:
            assert np.array_equal(np.asarray(got[k]).view(np.uint32) if got[k].dtype == np.float32 else got[k],
                                  d["exp_" + k].view(np.uint32) if d["exp_" + k].dtype == np.float32 else d["exp_" + k]), (f, k)


def test_empty_legal_list_is_every_action():
    """A root with an empty legal list (or an all-zero mask row) has every action legal, like CNode::expand, and takes the
    first A Gumbel draws: the same search as an explicit 0..A-1 list."""
    from lightzero_b200 import gmz_tree
    B, A, S, m = 3, 6, 16, 4
    rng = np.random.default_rng(5)
    logits = _q(rng, (B, A), 0.5).tolist()
    values = _q(rng, (B,), 0.25).tolist()
    outs = []
    for legal in ([[], [0, 2], []], [list(range(A)), [0, 2], list(range(A))],
                  np.array([[0] * A, [1, 0, 1, 0, 0, 0], [0] * A], np.uint8)):
        roots = gmz_tree.Roots(B, legal)
        roots.prepare_no_noise([0.0] * B, values, logits, [-1] * B)
        rec = []
        for sim in range(S):
            res = gmz_tree.ResultsWrapper(B)
            ix, iy, la, vtp = gmz_tree.batch_traverse(roots, S, m, 0.997, res, [-1] * B)
            assert min(la) >= 0
            rec.append((ix, la, res.get_search_len()))
            gmz_tree.batch_back_propagate(sim + 1, 0.997, _q(rng, (B,), 0.5).tolist(), _q(rng, (B,), 0.25).tolist(),
                                          _q(rng, (B, A), 1.0).tolist(), None, res, vtp)
        outs.append((rec, roots.get_distributions(), _bits(roots.get_policies(0.997, A)).tolist()))
        roots.clear()
        rng = np.random.default_rng(5)
        rng.normal(size=B * A + B)       # same synthetic stream for each legal form
    assert outs[0] == outs[1] == outs[2]
    assert all(len(d) == A for d in (outs[0][1][0], outs[0][1][2]))


def test_refusals():
    from lightzero_b200 import cabi
    lib = cabi.load()
    B, A, S = 4, 6, 3
    h = ctypes.c_void_p()
    cabi.check(lib.lz_tree_create(B, A, S, h), "lz_tree_create")
    try:
        dev = torch.device("cuda")
        logits = torch.zeros(B, A, device=dev)
        vals = torch.zeros(B, device=dev)
        i32 = [torch.zeros(B, dtype=torch.int32, device=dev) for _ in range(5)]
        s = cabi.stream_ptr()
        cabi.check(lib.lz_tree_set_gumbel(h, A, S), "lz_tree_set_gumbel")
        assert lib.lz_tree_set_ez(h, 1, 5) < 0
        cabi.check(lib.lz_tree_reset(h, None, None, s), "lz_tree_reset")
        assert lib.lz_tree_traverse_gumbel(h, *[t.data_ptr() for t in i32], s) < 0      # not prepared
        cabi.check(lib.lz_tree_prepare_gumbel(h, logits.data_ptr(), None, 0.0, None, vals.data_ptr(), None, s), "prepare")
        assert lib.lz_tree_traverse(h, 1, *[t.data_ptr() for t in i32], s) < 0           # MuZero call on a Gumbel tree
        assert lib.lz_tree_backpropagate_gumbel(h, 1, vals.data_ptr(), vals.data_ptr(), logits.data_ptr(), None, s) < 0
        for sim in range(S):
            cabi.check(lib.lz_tree_traverse_gumbel(h, *[t.data_ptr() for t in i32], s), "traverse")
            cabi.check(lib.lz_tree_backpropagate_gumbel(h, sim + 1, vals.data_ptr(), vals.data_ptr(), logits.data_ptr(), None, s), "bp")
        rc = lib.lz_tree_traverse_gumbel(h, *[t.data_ptr() for t in i32], s)                # one past num_simulations
        assert rc < 0 and b"considered-visit table" in lib.lz_last_error()
        torch.cuda.synchronize()
        cabi.check(lib.lz_tree_set_gumbel(h, 0, 0), "lz_tree_set_gumbel off")
        cabi.check(lib.lz_tree_set_ez(h, 1, 5), "lz_tree_set_ez")
        assert lib.lz_tree_set_gumbel(h, A, S) < 0                                        # EfficientZero tree
    finally:
        lib.lz_tree_destroy(h)
    import lightzero_b200 as lzb
    mcts = lzb.GumbelMuZeroMCTSCtree(dict(num_simulations=2))
    with pytest.raises(TypeError):
        mcts.search(mcts.roots(1, [[0, 1]]), lzb.EfficientZeroModel.__new__(lzb.EfficientZeroModel), np.zeros((1, 64, 6, 6)), [-1])
