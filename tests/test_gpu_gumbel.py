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

from oracle.tree_drive import Sampled, assert_same, check_fixture, drive, network, readout

pytestmark = pytest.mark.gpu


def _oracle():
    from oracle import build_gmz_ref
    mod = build_gmz_ref.load()
    if mod is None:
        pytest.skip("compiled reference Gumbel tree not built (oracle/build_gmz_ref.py)")
    return mod


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


def _case(B, A, S, m, legal, seed, noise, to_play):
    """Synthetic inputs and network outputs (quantised so that scores tie): root logits, values and noise, then per
    simulation reward, value and policy logits drawn by the returned Sampled source."""
    rng = np.random.default_rng(seed)
    c = dict(B=B, A=A, S=S, m=m, legal=legal, to_play=to_play, noise=int(noise), root_logits=_q(rng, (B, A), 0.5),
             root_values=_q(rng, (B,), 0.25))
    if noise:
        c["noises"] = [rng.dirichlet([0.3] * len(l)).astype(np.float32).tolist() for l in legal]
    return c, Sampled(lambda: (_q(rng, (B,), 0.5), _q(rng, (B,), 0.25), _q(rng, (B, A), 1.0)))


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
    c, leaves = _case(B, A, S, m, legal, seed, noise, to_play)
    exp, _ = drive(ref, c, "gumbel", leaves)
    c, leaves = _case(B, A, S, m, legal, seed, noise, to_play)
    got, roots = drive(gmz_tree, c, "gumbel", leaves)
    assert_same(got, exp)
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


def _oracle_search(ref, model, out, legal, noises, B, A, S, m):
    """The reference tree picks every leaf, the CUDA network evaluates it (recurrent_inference(return_scalars=True))."""
    c = dict(B=B, A=A, S=S, m=m, legal=legal, to_play=-1, noises=noises, root_logits=out.policy_logits.cpu().numpy(),
             root_values=out.value_scalar.cpu().numpy())
    return drive(ref, c, "gumbel", network(model, out.latent_state))[0]


def _fused_search(model, out, legal, noises, B, A, S, m):
    import lightzero_b200 as lzb
    mcts = lzb.GumbelMuZeroMCTSCtree(dict(num_simulations=S, max_num_considered_actions=m))
    roots = mcts.roots(B, legal)
    roots.prepare(0.25, noises, [0.0] * B, out.value_scalar, out.policy_logits, [-1] * B)
    mcts.search(roots, model, out.latent_state, [-1] * B)
    return readout(roots, A, S, 0.997), mcts, roots


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
    assert_same(got, _oracle_search(ref, model, out, legal, noises, B, A, S, m))
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
    assert_same(fused, readout(roots2, A, S, 0.997))
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
        assert_same(got, _oracle_search(ref, model, out, legal, noises, B, A, S, mm_))
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
    _, files = _golden()
    for f in files:
        _, roots = check_fixture(gmz_tree, np.load(f))
        roots.clear()


def test_empty_legal_list_is_every_action():
    """A root with an empty legal list (or an all-zero mask row) has every action legal, like CNode::expand, and takes the
    first A Gumbel draws: the same search as an explicit 0..A-1 list."""
    from lightzero_b200 import gmz_tree
    B, A, S, m = 3, 6, 16, 4
    rng = np.random.default_rng(5)
    c = dict(B=B, A=A, S=S, m=m, to_play=-1, root_logits=_q(rng, (B, A), 0.5), root_values=_q(rng, (B,), 0.25))
    outs = []
    for legal in ([[], [0, 2], []], [list(range(A)), [0, 2], list(range(A))],
                  np.array([[0] * A, [1, 0, 1, 0, 0, 0], [0] * A], np.uint8)):
        rng = np.random.default_rng(5)
        rng.normal(size=B * A + B)       # same synthetic stream for each legal form
        t, roots = drive(gmz_tree, dict(c, legal=legal), "gumbel",
                         Sampled(lambda: (_q(rng, (B,), 0.5), _q(rng, (B,), 0.25), _q(rng, (B, A), 1.0))))
        roots.clear()
        assert (t["last_action"] >= 0).all()
        outs.append({k: t[k] for k in ("ix", "last_action", "search_len", "distributions", "policies")})
    assert_same(outs[1], outs[0])
    assert_same(outs[2], outs[0])
    assert (outs[0]["distributions"][[0, 2]] >= 0).all()


def test_tree_entry_point_refusals():
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
        leaves = [t.data_ptr() for t in i32] + [None]       # ix, iy, last action, search length, virtual to_play; no is_reset
        s = cabi.stream_ptr()
        cabi.check(lib.lz_tree_set_gumbel(h, A, S), "lz_tree_set_gumbel")
        assert lib.lz_tree_set_ez(h, 1, 5) < 0
        cabi.check(lib.lz_tree_reset(h, None, None, s), "lz_tree_reset")
        assert lib.lz_tree_traverse(h, 1, None, None, *leaves, s) < 0                       # not prepared
        assert lib.lz_tree_prepare(h, logits.data_ptr(), None, 0.0, None, None, None, s) < 0   # Gumbel roots need their values
        cabi.check(lib.lz_tree_prepare(h, logits.data_ptr(), None, 0.0, None, vals.data_ptr(), None, s), "prepare")
        ta = torch.zeros(B, dtype=torch.int32, device=dev)
        assert lib.lz_tree_traverse(h, 1, ta.data_ptr(), vals.data_ptr(), *leaves, s) < 0   # reuse descent on a Gumbel tree
        no_bp = lib.lz_tree_backpropagate(h, 1, vals.data_ptr(), vals.data_ptr(), logits.data_ptr(), None, None, None, None, s)
        assert no_bp < 0                                                                  # back-up before any descent
        for sim in range(S):
            cabi.check(lib.lz_tree_traverse(h, 1, None, None, *leaves, s), "traverse")
            cabi.check(lib.lz_tree_backpropagate(h, sim + 1, vals.data_ptr(), vals.data_ptr(), logits.data_ptr(), None, None, None,
                                                 None, s), "bp")
        rc = lib.lz_tree_traverse(h, 1, None, None, *leaves, s)                             # one past num_simulations
        assert rc < 0 and b"considered-visit table" in lib.lz_last_error()
        torch.cuda.synchronize()
        cabi.check(lib.lz_tree_set_gumbel(h, 0, 0), "lz_tree_set_gumbel off")
        assert lib.lz_tree_prepare(h, logits.data_ptr(), None, 0.0, None, vals.data_ptr(), None, s) == -1   # values: Gumbel only
        assert lib.lz_tree_traverse(h, 1, None, None, *leaves[:5], i32[0].data_ptr(), s) == -1    # is_reset: EfficientZero only
        assert lib.lz_tree_traverse(h, 1, ta.data_ptr(), None, *leaves, s) == -1                # half a reuse pair
        assert lib.lz_tree_backpropagate(h, 1, vals.data_ptr(), vals.data_ptr(), logits.data_ptr(), None, ta.data_ptr(), None,
                                         None, s) == -1                                         # batch rank without reuse
        cabi.check(lib.lz_tree_set_ez(h, 1, 5), "lz_tree_set_ez")
        assert lib.lz_tree_set_gumbel(h, A, S) < 0                                        # EfficientZero tree
        assert lib.lz_tree_backpropagate(h, 1, vals.data_ptr(), vals.data_ptr(), logits.data_ptr(), None, None, None, None,
                                         s) == -1                                               # EfficientZero needs is_reset
    finally:
        lib.lz_tree_destroy(h)
    import lightzero_b200 as lzb
    mcts = lzb.GumbelMuZeroMCTSCtree(dict(num_simulations=2))
    with pytest.raises(TypeError):
        mcts.search(mcts.roots(1, [[0, 1]]), lzb.EfficientZeroModel.__new__(lzb.EfficientZeroModel), np.zeros((1, 64, 6, 6)), [-1])
