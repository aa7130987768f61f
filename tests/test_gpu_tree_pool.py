"""Pooled trees handed from one entry point to the next (mz_tree.acquire_tree, TreeHandle.set_mode).

A pooled tree's mode (MuZero, EfficientZero, Gumbel) and tie rule are C state that outlives its holder; every acquirer sets
all of it once.  These tests check that nothing a holder set carries over to the next one, and that setting the mode on
every acquisition re-captures no search graph."""
import contextlib

import numpy as np
import pytest
import torch

from oracle.tree_drive import assert_same, drive, recorded
from test_oracle_tie_hash import port_drive, tie_rich_case

pytestmark = pytest.mark.gpu

OBS = (4, 84, 84)


def _model(A, ez=False):
    import lightzero_b200 as lzb
    from lightzero_b200.synthetic_weights import synthetic_state_dict
    cls = lzb.EfficientZeroModel if ez else lzb.MuZeroModel
    return cls(observation_shape=OBS, action_space_size=A).load_state_dict(synthetic_state_dict(OBS, A, efficientzero=ez, seed=3))


def _inputs(B, A, seed):
    rng = np.random.default_rng(seed)
    obs = torch.from_numpy(rng.random((B,) + OBS, dtype=np.float32)).cuda()
    noise = rng.dirichlet([0.3] * A, size=B).astype(np.float32)
    return obs, noise


def _search(mcts, model, obs, noise, legal=None, reuse=False):
    """One MCTS search on fresh roots from the model's initial inference; returns (visits, values) and clears the roots."""
    B, A = noise.shape
    out = model.initial_inference(obs)
    roots = mcts.roots(B, legal or [list(range(A))] * B)
    roots.prepare(0.25, noise.tolist(), [0.] * B, out.policy_logits, [-1] * B)
    hidden = (out.reward_hidden_state,) if hasattr(out, "reward_hidden_state") else ()
    if reuse:
        mcts.search_with_reuse(roots, model, out.latent_state, *hidden, [-1] * B, [l[0] for l in roots._legal_lists], [0.5] * B)
    else:
        mcts.search(roots, model, out.latent_state, *hidden, [-1] * B)
    res = (roots.get_distributions(), np.asarray(roots.get_values(), np.float32))
    roots.clear()
    return res


def _captures():
    from lightzero_b200 import cabi
    return cabi.load().lz_debug_graph_captures()


# ------------------------------------------------------------------------------------------------ the tie rule does not leak
@pytest.mark.parametrize("kind", ["ez", "reuse"])
def test_stochastic_search_leaves_first_maximum_to_the_next_roots(kind):
    """A deterministic=False fused search (EfficientZero search, MuZero search_with_reuse) draws its ties; the step-wise mirror
    Roots that acquire its pooled tree next take the first maximum, as ez_tree / mz_tree document: the tie-rich drive equals
    the first-maximum C port."""
    import lightzero_b200 as lzb
    from lightzero_b200 import ez_tree, mz_tree
    B, A, S = 40, 7, 30
    c = tie_rich_case(B, A, S, 611 + len(kind))
    ez = kind == "ez"
    model = _model(A, ez=ez)
    obs, noise = _inputs(B, A, 5)
    cls = lzb.EfficientZeroMCTSCtree if ez else lzb.MuZeroMCTSCtree
    _search(cls(dict(num_simulations=S, deterministic=False)), model, obs, noise, reuse=not ez)
    got, roots = drive(ez_tree if ez else mz_tree, c, kind, recorded(c, kind))
    roots.clear()
    assert_same(got, port_drive(kind, c, det=True)[0])


# ------------------------------------------------------------------------------------------------ no extra graph captures
def _assert_no_recapture(call):
    call()
    n0 = _captures()
    for _ in range(3):
        call()
    assert _captures() == n0, "a repeated call re-captured a search graph"


@pytest.mark.parametrize("det", [False, True])
@pytest.mark.parametrize("ez", [False, True])
def test_repeated_search_captures_no_graph(ez, det):
    import lightzero_b200 as lzb
    B, A, S = 24, 6, 12
    model = _model(A, ez=ez)
    obs, noise = _inputs(B, A, 7)
    mcts = (lzb.EfficientZeroMCTSCtree if ez else lzb.MuZeroMCTSCtree)(dict(num_simulations=S, deterministic=det))
    _assert_no_recapture(lambda: _search(mcts, model, obs, noise))


def test_search_alternating_with_reuse_captures_no_graph():
    """ReZero's own loop on one deterministic=False MuZero tree: search, then search_with_reuse, over and over."""
    import lightzero_b200 as lzb
    B, A, S = 24, 6, 12
    model = _model(A)
    obs, noise = _inputs(B, A, 8)
    mcts = lzb.MuZeroMCTSCtree(dict(num_simulations=S, deterministic=False))
    _assert_no_recapture(lambda: (_search(mcts, model, obs, noise), _search(mcts, model, obs, noise, reuse=True)))


def test_repeated_gumbel_search_captures_no_graph():
    import lightzero_b200 as lzb
    B, A, S = 24, 6, 12
    model = _model(A)
    obs, noise = _inputs(B, A, 9)
    mcts = lzb.GumbelMuZeroMCTSCtree(dict(num_simulations=S, max_num_considered_actions=4))

    def call():
        out = model.initial_inference(obs, return_scalar_value=True)
        roots = mcts.roots(B, [list(range(A))] * B)
        roots.prepare(0.25, noise.tolist(), [0.] * B, out.value_scalar, out.policy_logits, [-1] * B)
        mcts.search(roots, model, out.latent_state, [-1] * B)
        roots.get_distributions()
        roots.clear()
    _assert_no_recapture(call)


@pytest.mark.parametrize("policy", ["MuZeroCollectPolicy", "EfficientZeroCollectPolicy", "GumbelMuZeroCollectPolicy"])
def test_repeated_collect_captures_no_graph(policy):
    import lightzero_b200 as lzb
    B, A, S = 24, 6, 12
    model = _model(A, ez=policy.startswith("Eff"))
    obs, noise = _inputs(B, A, 10)
    pol = getattr(lzb, policy)(model, dict(num_simulations=S, deterministic=False))
    mask = np.ones((B, A), np.uint8)
    _assert_no_recapture(lambda: pol.search_batch(obs, mask, noise, select=(1.0, False, 0)))


# ------------------------------------------------------------------------------------------------ pool hand-over
class _Stepwise:
    """Any model object that is not a lightzero_b200 model: the search drives the device tree one simulation at a time."""

    def __init__(self, model):
        self.model = model

    def initial_inference(self, *args):
        return self.model.initial_inference(*args)

    def recurrent_inference(self, *args):
        return self.model.recurrent_inference(*args)


@contextlib.contextmanager
def _fresh_tree(B, A, S):
    """Holds every pooled tree of this shape, so that the next acquirer of the shape gets a new tree."""
    from lightzero_b200 import mz_tree
    dev = torch.device("cuda", torch.cuda.current_device())
    held = []
    while any(not h.busy for h in mz_tree._tree_pool.get((dev.index, B, A, S), [])):
        held.append(mz_tree.acquire_tree(dev, B, A, S))
    try:
        yield
    finally:
        for h in held:
            h.release()


def test_pool_hand_over_between_entry_points():
    """One pooled shape used by a MuZero collect, a Gumbel collect, a step-wise EfficientZero search and a fused MuZero
    search, in that order: each result equals the same call on a new tree."""
    import lightzero_b200 as lzb
    B, A, S = 20, 6, 14
    mz, ez = _model(A), _model(A, ez=True)
    obs, noise = _inputs(B, A, 12)
    mask = np.ones((B, A), np.uint8)
    mz_collect = lzb.MuZeroCollectPolicy(mz, dict(num_simulations=S, deterministic=True))
    gumbel_collect = lzb.GumbelMuZeroCollectPolicy(mz, dict(num_simulations=S, max_num_considered_actions=4))
    ez_search = lzb.EfficientZeroMCTSCtree(dict(num_simulations=S))
    mz_search = lzb.MuZeroMCTSCtree(dict(num_simulations=S, deterministic=True))

    def collect(pol):
        r = pol.search_batch(obs, mask, noise, select=(1.0, False, 0))
        return {k: v.clone() for k, v in r.items()}
    calls = [lambda: collect(mz_collect), lambda: collect(gumbel_collect),
             lambda: _search(ez_search, _Stepwise(ez), obs, noise), lambda: _search(mz_search, mz, obs, noise)]
    handed = [call() for call in calls]
    for call, got in zip(calls, handed):
        with _fresh_tree(B, A, S):
            exp = call()
        if isinstance(got, dict):
            assert got.keys() == exp.keys()
            for k in got:
                assert torch.equal(got[k], exp[k]), k
        else:
            assert got[0] == exp[0]
            assert np.array_equal(got[1].view(np.uint32), exp[1].view(np.uint32))
