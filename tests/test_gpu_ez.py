"""GPU parity tests of the EfficientZero path (SURVEY.md 8(f) row f-1 / BASELINE config 2): the CUDA EfficientZeroModel
against vectors produced by the reference's own model class and against the PyTorch restatement live, and the fused
EfficientZeroMCTSCtree search against the step-wise drive, the oracle pipeline replay and the oracle pipeline end to end.
Also: every model fixture (MuZero, EfficientZero, MLP) through the corresponding CUDA model."""
import glob
import os
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN_DIR, ROOT

pytestmark = pytest.mark.gpu
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))

MODEL_CASES = sorted(os.path.basename(p)[:-4] for p in glob.glob(os.path.join(GOLDEN_DIR, "model_*.npz")))
TOL = dict(rtol=1e-5, atol=1e-5)        # the 1e-5 fp32 bar of the north star (logits, latents, LSTM state)


def _cuda_model_for(kind, obs_shape, A, nres, state_dict):
    import lightzero_b200 as lzb
    if kind == "muzero":
        return lzb.MuZeroModel(observation_shape=obs_shape, action_space_size=A, num_res_blocks=nres).load_state_dict(state_dict)
    if kind == "efficientzero":
        return lzb.EfficientZeroModel(observation_shape=obs_shape, action_space_size=A, num_res_blocks=nres).load_state_dict(state_dict)
    return lzb.MuZeroModelMLP(observation_shape=obs_shape, action_space_size=A, latent_state_dim=128,
                              res_connection_in_dynamics=True).load_state_dict(state_dict)


@pytest.mark.parametrize("name", MODEL_CASES)
def test_cuda_model_matches_reference_class_vectors(name):
    """Fixtures written by tests/golden/make_model_golden.py from the REFERENCE'S OWN model classes; the weights are
    regenerated from the fixture's seed through the restatement (checked by SHA-256)."""
    from make_model_golden import build_restated, weights_digest
    d = np.load(os.path.join(GOLDEN_DIR, name + ".npz"))
    kind = str(d["kind"])
    obs_shape = int(d["obs_shape"]) if d["obs_shape"].ndim == 0 else tuple(int(x) for x in d["obs_shape"])
    ref = build_restated(kind, obs_shape, int(d["A"]), int(d["nres"]), int(d["seed"]))
    if weights_digest(ref) != str(d["weights_sha256"]):
        pytest.skip("this torch build initialises parameters differently from the one that wrote the fixture")
    cu = _cuda_model_for(kind, obs_shape, int(d["A"]), int(d["nres"]), ref.state_dict())
    obs, action = torch.from_numpy(d["obs"]).cuda(), torch.from_numpy(d["action"]).cuda()
    o0 = cu.initial_inference(obs)
    for f in ("value", "policy_logits", "latent_state"):
        assert torch.allclose(getattr(o0, f).cpu(), torch.from_numpy(d["init_" + f]), **TOL), (name, "initial", f)
    latent = torch.from_numpy(d["init_latent_state"]).cuda()
    if kind == "efficientzero":
        hc = (torch.from_numpy(d["in_hidden0"]).cuda(), torch.from_numpy(d["in_hidden1"]).cuda())
        o1 = cu.recurrent_inference(latent, hc, action)
        for f in ("value", "value_prefix", "policy_logits", "latent_state"):
            assert torch.allclose(getattr(o1, f).cpu(), torch.from_numpy(d["rec_" + f]), **TOL), (name, "recurrent", f)
        for i in range(2):
            assert o1.reward_hidden_state[i].shape == (1, obs.shape[0], 512)
            assert torch.allclose(o1.reward_hidden_state[i].cpu(), torch.from_numpy(d[f"rec_hidden{i}"]), **TOL), (name, "hidden", i)
    else:
        o1 = cu.recurrent_inference(latent, action)
        for f in ("value", "reward", "policy_logits", "latent_state"):
            assert torch.allclose(getattr(o1, f).cpu(), torch.from_numpy(d["rec_" + f]), **TOL), (name, "recurrent", f)


def _setup(B, A, S, seed=0, masks=False, horizon=5):
    import lightzero_b200 as lzb
    from oracle.model_ref import EfficientZeroModelRef, emulate_trained_
    torch.manual_seed(seed)
    ref = emulate_trained_(EfficientZeroModelRef((4, 96, 96), A), seed)
    cu = lzb.EfficientZeroModel(observation_shape=(4, 96, 96), action_space_size=A).load_state_dict(ref.state_dict())
    rng = np.random.default_rng(seed)
    obs = torch.rand(B, 4, 96, 96)
    mask = np.ones((B, A), np.uint8)
    if masks:
        mask = (rng.random((B, A)) < 0.6).astype(np.uint8)
        mask[np.arange(B), rng.integers(0, A, B)] = 1
    legal = [np.nonzero(mask[b])[0].tolist() for b in range(B)]
    noises = [rng.dirichlet([0.3] * len(l)).astype(np.float32).tolist() for l in legal]
    mcts = lzb.EfficientZeroMCTSCtree(dict(num_simulations=S, discount_factor=0.997, lstm_horizon_len=horizon))
    return ref, cu, obs, mask, legal, noises, mcts


@pytest.mark.parametrize("B", [7, 256, 1024])
def test_cuda_ez_model_matches_restatement_live(B):
    """Batch sizes up to the BASELINE sizes against the PyTorch restatement (itself pinned to the reference class)."""
    A = 6
    ref, cu, obs, *_ = _setup(min(B, 64), A, 1, seed=B)
    g = torch.Generator().manual_seed(B)
    latent = torch.rand(B, 64, 6, 6, generator=g) * 2
    hc = (torch.randn(1, B, 512, generator=g) * 0.5, torch.randn(1, B, 512, generator=g) * 0.5)
    action = torch.randint(0, A, (B,), generator=g)
    with torch.no_grad():
        exp = ref.recurrent_inference(latent, hc, action)
    got = cu.recurrent_inference(latent.cuda(), (hc[0].cuda(), hc[1].cuda()), action.cuda(), return_scalars=True)
    for f in ("value", "value_prefix", "policy_logits", "latent_state"):
        assert torch.allclose(getattr(got, f).cpu(), getattr(exp, f), **TOL), f
    for i in range(2):
        assert torch.allclose(got.reward_hidden_state[i].cpu(), exp.reward_hidden_state[i], **TOL), i
    from oracle.model_ref import DiscreteSupport, InverseScalarTransform
    inv = InverseScalarTransform(DiscreteSupport(-300., 301., 1.))
    # scalar outputs: the reference's own h^-1 is quantised in ~1.2e-4 steps near 0 (DESIGN.md 4.4)
    assert torch.allclose(got.value_prefix_scalar.cpu(), inv(exp.value_prefix).reshape(-1), rtol=0, atol=2e-4)
    assert torch.allclose(got.value_scalar.cpu(), inv(exp.value).reshape(-1), rtol=0, atol=2e-4)


class _Proxy:
    """Not an EfficientZeroModel instance -> the mirror drives the device trees one simulation at a time around it."""

    def __init__(self, model):
        self.model = model

    def eval(self):
        return self

    def recurrent_inference(self, latent, hidden, action):
        return self.model.recurrent_inference(latent, hidden, action)


@pytest.mark.parametrize("B,A,S,masks,horizon", [(16, 6, 20, False, 5), (256, 6, 50, False, 5), (130, 18, 40, True, 2)])
def test_fused_ez_search_equals_stepwise_search(B, A, S, masks, horizon):
    """One CUDA graph for the whole search vs the step-wise drive of the same kernels through the public pieces
    (lz_tree_traverse_ez / recurrent_inference / lz_tree_backpropagate_ez): identical visit counts and root value bits."""
    ref, cu, obs, mask, legal, noises, mcts = _setup(B, A, S, masks=masks, horizon=horizon)
    out = cu.initial_inference(obs.cuda())
    results = []
    for mode in ("fused", "fused", "step"):
        roots = mcts.roots(B, legal)
        roots.prepare(0.25, noises, [0.] * B, out.policy_logits, [-1] * B)
        mcts.search(roots, cu if mode != "step" else _Proxy(cu), out.latent_state, out.reward_hidden_state, [-1] * B)
        results.append((roots.get_distributions(), np.asarray(roots.get_values(), np.float32).view(np.uint32).tolist()))
        roots.clear()
    assert results[0] == results[1] == results[2]
    assert all(sum(d) == S for d in results[0][0])
    assert mcts.last_num_kernels == 1 + 4 * S        # traverse + S x (conv trunk, LSTM GEMM, value-prefix head, back-up)


def test_replay_of_reference_ez_pipeline_is_bit_exact():
    """Feed the CUDA value-prefix trees the network outputs recorded from the ORACLE pipeline (compiled
    ctree_efficientzero + PyTorch-CPU EfficientZero model): visit counts and root values must match bit for bit."""
    from lightzero_b200 import ez_tree, mz_tree
    from oracle.search_ref import SearchRefEZ, collect_step_ref_ez, load_tree_module
    B, A, S, H = 40, 18, 40, 3
    ref, cu, obs, mask, legal, noises, mcts = _setup(B, A, S, seed=5, masks=True, horizon=H)
    tree, kind = load_tree_module(name="ez_tree")
    rec = []
    exp = collect_step_ref_ez(SearchRefEZ(tree, lstm_horizon_len=H, num_simulations=S), ref, obs, mask, [-1] * B, noises=noises, recorder=rec)
    mz_tree.DEFAULT_MAX_SIMS = max(mz_tree.DEFAULT_MAX_SIMS, S)
    roots = ez_tree.Roots(B, legal)
    roots.prepare(0.25, noises, [0.] * B, exp["policy_logits"].tolist(), [-1] * B)
    mm = ez_tree.MinMaxStatsList(B)
    mm.set_delta(0.01)
    for s in range(S):
        res = ez_tree.ResultsWrapper(B)
        ix, iy, la, vtp = ez_tree.batch_traverse(roots, 19652, 1.25, 0.997, mm, res, [-1] * B)
        assert ix == rec[s]["ix"] and la == rec[s]["last_action"] and res.get_search_len() == rec[s]["search_len"]
        ez_tree.batch_backpropagate(s + 1, 0.997, rec[s]["reward"], rec[s]["value"], rec[s]["policy"], mm, res, rec[s]["is_reset"], vtp)
    assert roots.get_distributions() == exp["distributions"]
    assert np.array_equal(np.asarray(roots.get_values(), np.float32).view(np.uint32),
                          np.asarray(exp["values"], np.float32).view(np.uint32))
    assert sum(sum(r["is_reset"]) for r in rec) > 0


@pytest.mark.parametrize("B,A,S,masks,horizon", [(48, 6, 25, False, 5), (64, 18, 40, True, 3)])
def test_ez_end_to_end_against_reference_pipeline(B, A, S, masks, horizon):
    """Whole EfficientZero path vs the oracle pipeline.  Independent fp32 networks (PUCT is discontinuous), so identity
    of the visit counts is asserted for the large majority of roots and root values at 1e-5 on those that match."""
    from oracle.search_ref import SearchRefEZ, collect_step_ref_ez, load_tree_module
    ref, cu, obs, mask, legal, noises, mcts = _setup(B, A, S, seed=3, masks=masks, horizon=horizon)
    tree, kind = load_tree_module(name="ez_tree")
    exp = collect_step_ref_ez(SearchRefEZ(tree, lstm_horizon_len=horizon, num_simulations=S), ref, obs, mask, [-1] * B, noises=noises)
    out = cu.initial_inference(obs.cuda())
    assert torch.allclose(out.policy_logits.cpu(), torch.from_numpy(exp["policy_logits"]), **TOL)
    roots = mcts.roots(B, legal)
    roots.prepare(0.25, noises, [0.] * B, out.policy_logits, [-1] * B)
    mcts.search(roots, cu, out.latent_state, out.reward_hidden_state, [-1] * B)
    got_d, got_v = roots.get_distributions(), roots.get_values()
    same = [g == e for g, e in zip(got_d, exp["distributions"])]
    print(f"identical visit distributions: {sum(same)}/{B} (tree oracle: {kind})")
    assert sum(same) / B >= 0.85
    for i in range(B):
        if same[i]:
            assert abs(got_v[i] - exp["values"][i]) <= 1e-5 + 2e-4 * abs(exp["values"][i])
    assert all(sum(d) == S for d in got_d)


def test_ez_search_rejects_mismatched_model_and_tree():
    import lightzero_b200 as lzb
    ref, cu, obs, mask, legal, noises, mcts = _setup(8, 6, 5)
    out = cu.initial_inference(obs.cuda())
    mz = lzb.MuZeroMCTSCtree(dict(num_simulations=5))
    roots = mz.roots(8, legal)
    roots.prepare(0.25, noises, [0.] * 8, out.policy_logits, [-1] * 8)
    with pytest.raises(TypeError):
        mz.search(roots, cu, out.latent_state, [-1] * 8)


def test_fused_ez_search_with_reuse_equals_piecewise_drive():
    """EfficientZeroMCTSCtree.search_with_reuse (mcts_ctree.py:878-1003) as one CUDA graph vs the same steps driven one at a time
    through the public pieces (lz_tree_traverse_with_reuse, EfficientZeroModel.recurrent_inference on every row,
    lz_tree_backpropagate_with_reuse with the per-tree is_reset): identical visit counts, value bits and inference counts.
    (The tree entry points themselves are pinned to the shimmed reference ez_tree in test_gpu_tree.py.)"""
    from lightzero_b200 import cabi
    B, A, S, H = 64, 6, 25, 3
    ref, cu, obs, mask, legal, noises, mcts = _setup(B, A, S, masks=True, horizon=H)
    out = cu.initial_inference(obs.cuda())
    rng = np.random.default_rng(4)
    true_action = [int(l[rng.integers(len(l))]) for l in legal]
    reuse_value = (rng.standard_normal(B) * 0.5).astype(np.float32)
    roots = mcts.roots(B, legal)
    roots.prepare(0.25, noises, [0.] * B, out.policy_logits, [-1] * B)
    length, avg = mcts.search_with_reuse(roots, cu, out.latent_state, out.reward_hidden_state, [-1] * B, true_action, reuse_value.tolist())
    fused = (roots.get_distributions(), np.asarray(roots.get_values(), np.float32).view(np.uint32).tolist())
    roots.clear()

    roots = mcts.roots(B, legal)
    roots.prepare(0.25, noises, [0.] * B, out.policy_logits, [-1] * B)
    roots._ez, roots._lstm_horizon = True, H
    roots._materialize(S, mcts._params())
    t = roots._tree
    dev = roots.device
    ta = torch.tensor(true_action, dtype=torch.int32, device=dev)
    rv = torch.from_numpy(reuse_value).to(dev)
    lat = out.latent_state
    pool = torch.empty((S + 1,) + tuple(lat.shape), device=dev)
    hp0, hp1 = torch.zeros(S + 1, B, 512, device=dev), torch.zeros(S + 1, B, 512, device=dev)
    pool[0], hp0[0], hp1[0] = lat, out.reward_hidden_state[0].reshape(B, -1), out.reward_hidden_state[1].reshape(B, -1)
    rows = torch.arange(B, device=dev)
    counts = []
    for sim in range(S):
        cabi.check(t.lib.lz_tree_traverse_with_reuse(t.h, ta.data_ptr(), rv.data_ptr(), t.ix.data_ptr(), t.iy.data_ptr(), t.action.data_ptr(),
                                                     t.search_len.data_ptr(), t.vtp.data_ptr(), cabi.stream_ptr()), "traverse")
        counts.append(int((t.ix >= 0).sum().item()))
        ix = t.ix.clamp(min=0).long()
        reset = (t.search_len % H == 0).to(torch.int32)
        o = cu.recurrent_inference(pool[ix, rows], (hp0[ix, rows].unsqueeze(0), hp1[ix, rows].unsqueeze(0)), t.action.clamp(min=0).long(),
                                   return_scalars=True)
        pool[sim + 1] = o.latent_state
        keep = (reset == 0).float().unsqueeze(1)
        hp0[sim + 1] = o.reward_hidden_state[0].reshape(B, -1) * keep
        hp1[sim + 1] = o.reward_hidden_state[1].reshape(B, -1) * keep
        cabi.check(t.lib.lz_tree_backpropagate_with_reuse(t.h, sim + 1, o.value_prefix_scalar.data_ptr(), o.value_scalar.data_ptr(),
                                                          o.policy_logits.data_ptr(), rv.data_ptr(), None, reset.data_ptr(), None,
                                                          cabi.stream_ptr()), "backprop")
    step = (roots.get_distributions(), np.asarray(roots.get_values(), np.float32).view(np.uint32).tolist())
    assert fused == step
    assert length == counts[-1] and abs(avg - sum(counts) / S) < 1e-9
    assert min(counts) < B
    # traverse + S x (conv trunk, LSTM GEMM, value-prefix head, back-up) + (S - 1) x traverse
    assert mcts.last_num_kernels == 5 * S


def test_ez_stochastic_tiebreak_is_legal_and_reproducible():
    """lz_tree_set_tiebreak(0) (config deterministic=False): the EfficientZero descent draws from the reference's tie list
    (ctree_efficientzero/lib/cnode.cpp:676-691) with the counter-based device RNG: searches stay legal (sum of visits = S, masked actions
    never visited) and differ from the first-maximum search only where ties exist (all-equal priors and zero values force ties at the root)."""
    import lightzero_b200 as lzb
    B, A, S = 32, 6, 12
    ref, cu, obs, mask, legal, noises, mcts = _setup(B, A, S, masks=True, horizon=3)
    out = cu.initial_inference(obs.cuda())
    flat = torch.zeros_like(out.policy_logits)                 # equal priors: every first descent is a tie
    res = {}
    for det in (True, False):
        m = lzb.EfficientZeroMCTSCtree(dict(num_simulations=S, discount_factor=0.997, lstm_horizon_len=3, deterministic=det))
        roots = m.roots(B, legal)
        roots.prepare_no_noise([0.] * B, flat, [-1] * B)
        m.search(roots, cu, out.latent_state, out.reward_hidden_state, [-1] * B)
        res[det] = roots.get_distributions()
        assert all(sum(d) == S and len(d) == len(l) for d, l in zip(res[det], legal))
        roots.clear()
    assert res[True] != res[False]
