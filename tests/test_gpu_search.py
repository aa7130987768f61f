"""GPU tests of the fused search (one CUDA graph per search) through the MuZeroMCTSCtree mirror."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _setup(B, A, S, seed=0, masks=False, math=None):
    import lightzero_b200 as lzb
    from oracle.model_ref import MuZeroModelRef, emulate_trained_
    torch.manual_seed(seed)
    ref = emulate_trained_(MuZeroModelRef((4, 84, 84), A), seed)
    cu = lzb.MuZeroModel(observation_shape=(4, 84, 84), action_space_size=A).load_state_dict(ref.state_dict())
    if math is not None:
        cu.set_math(math)
    rng = np.random.default_rng(seed)
    obs = torch.rand(B, 4, 84, 84)
    mask = np.ones((B, A), np.uint8)
    if masks:
        mask = (rng.random((B, A)) < 0.6).astype(np.uint8)
        mask[np.arange(B), rng.integers(0, A, B)] = 1
    legal = [np.nonzero(mask[b])[0].tolist() for b in range(B)]
    noises = [rng.dirichlet([0.3] * len(l)).astype(np.float32).tolist() for l in legal]
    mcts = lzb.MuZeroMCTSCtree(dict(num_simulations=S, deterministic=True, discount_factor=0.997))
    return ref, cu, obs, mask, legal, noises, mcts


class _Recorder:
    """Wraps the CUDA model so the step-wise search records what the network returned."""

    def __init__(self, model):
        self.model, self.calls = model, []

    def eval(self):
        return self

    def recurrent_inference(self, latent, action):
        out = self.model.recurrent_inference(latent, action)
        self.calls.append((latent.clone(), action.clone(), out))
        return out


@pytest.mark.parametrize("math", ["tc3", "tc1"])
@pytest.mark.parametrize("B,A,S,masks", [(16, 6, 20, False), (300, 18, 50, True), (1024, 6, 50, False), (64, 40, 20, True)])
def test_fused_graph_search_equals_stepwise_search(B, A, S, masks, math):
    """The single-graph search and the one-simulation-at-a-time drive of the same kernels must agree
    exactly: visit counts, root values (bits), and repeated graph launches must be reproducible."""
    ref, cu, obs, mask, legal, noises, mcts = _setup(B, A, S, masks=masks, math=math)
    out = cu.initial_inference(obs.cuda())
    results = []
    for mode in ("fused", "fused", "step"):
        roots = mcts.roots(B, legal)
        roots.prepare(0.25, noises, [0.] * B, out.policy_logits, [-1] * B)
        mcts.search(roots, cu if mode != "step" else _Recorder(cu), out.latent_state, [-1] * B)
        results.append((roots.get_distributions(), np.asarray(roots.get_values(), np.float32).view(np.uint32).tolist()))
        roots.clear()
    assert results[0] == results[1] == results[2]
    assert all(sum(d) == S for d in results[0][0])
    # tensor-core path with A <= 32: one persistent launch; else [traverse] + S x [network, backprop(+traverse)] kernels
    assert mcts.last_num_kernels == (1 if A <= 32 else 2 * S + 1)


def test_search_accepts_numpy_latents_and_host_lists():
    """The reference passes latent_state_roots as np.ndarray and policy logits as nested lists
    (policy/muzero.py:757-758,774-775); the mirror must take exactly that."""
    B, A, S = 12, 6, 10
    ref, cu, obs, mask, legal, noises, mcts = _setup(B, A, S)
    out = cu.initial_inference(obs.cuda())
    roots = mcts.roots(B, legal)
    roots.prepare(0.25, noises, [0.] * B, out.policy_logits.cpu().numpy().tolist(), [-1] * B)
    mcts.search(roots, cu, out.latent_state.cpu().numpy(), [-1] * B)
    a = roots.get_distributions()
    roots2 = mcts.roots(B, legal)
    roots2.prepare(0.25, noises, [0.] * B, out.policy_logits, [-1] * B)
    mcts.search(roots2, cu, out.latent_state, [-1] * B)
    assert a == roots2.get_distributions()
    assert len(a) == B and all(len(d) == A for d in a) and isinstance(roots.get_values()[0], float)


@pytest.mark.parametrize("math", ["tc3"])
@pytest.mark.parametrize("B,A,S,masks", [(64, 6, 25, False), (96, 18, 50, True), (128, 18, 30, True), (48, 40, 20, True)])
def test_end_to_end_against_reference_pipeline(B, A, S, masks, math):
    """Whole path vs the oracle pipeline (PyTorch-CPU fp32 model + reference ctree, deterministic).
    Network outputs agree to ~1e-6, but PUCT is discontinuous (a flipped arg-max changes every later
    simulation of that root), so identity of visit counts is asserted per root for the large majority
    and the trees that do match must have root values within 1e-5."""
    from oracle.search_ref import SearchRef, collect_step_ref, load_tree_module
    ref, cu, obs, mask, legal, noises, mcts = _setup(B, A, S, seed=3, masks=masks, math=math)
    tree, kind = load_tree_module()
    sref = SearchRef(tree, num_simulations=S)
    exp = collect_step_ref(sref, ref, obs, mask, [-1] * B, noises=noises)
    out = cu.initial_inference(obs.cuda())
    assert torch.allclose(out.policy_logits.cpu(), torch.from_numpy(exp["policy_logits"]), rtol=1e-5, atol=1e-5)
    roots = mcts.roots(B, legal)
    roots.prepare(0.25, noises, [0.] * B, out.policy_logits, [-1] * B)
    mcts.search(roots, cu, out.latent_state, [-1] * B)
    got_d, got_v = roots.get_distributions(), roots.get_values()
    same = [g == e for g, e in zip(got_d, exp["distributions"])]
    frac = sum(same) / B
    print(f"identical visit distributions: {sum(same)}/{B} (tree oracle: {kind})")
    assert frac >= 0.85, frac
    for i in range(B):
        if same[i]:
            assert abs(got_v[i] - exp["values"][i]) <= 1e-5 + 2e-4 * abs(exp["values"][i])
    assert all(sum(d) == S for d in got_d)


@pytest.mark.parametrize("B,A,S", [(48, 18, 50), (128, 18, 200)])
def test_replay_of_reference_pipeline_is_bit_exact(B, A, S):
    """Replay mode (SURVEY.md s.7): feed the CUDA trees the network outputs the ORACLE pipeline
    produced (recorded per simulation).  The trees must then reproduce the reference's visit counts
    and root values bit for bit, on the same seeds -- also at BASELINE config 3's 200 simulations on a 128-root shard."""
    from lightzero_b200 import mz_tree
    from oracle.search_ref import SearchRef, collect_step_ref, load_tree_module
    ref, cu, obs, mask, legal, noises, mcts = _setup(B, A, S, seed=5, masks=True)
    tree, kind = load_tree_module()
    rec = []
    exp = collect_step_ref(SearchRef(tree, num_simulations=S), ref, obs, mask, [-1] * B, noises=noises, recorder=rec)
    mz_tree.DEFAULT_MAX_SIMS = max(mz_tree.DEFAULT_MAX_SIMS, S)
    roots = mz_tree.Roots(B, legal)
    roots.prepare(0.25, noises, [0.] * B, exp["policy_logits"].tolist(), [-1] * B)
    mm = mz_tree.MinMaxStatsList(B)
    mm.set_delta(0.01)
    for s in range(S):
        res = mz_tree.ResultsWrapper(B)
        ix, iy, la, vtp = mz_tree.batch_traverse(roots, 19652, 1.25, 0.997, mm, res, [-1] * B, True)
        assert ix == rec[s]["ix"] and la == rec[s]["last_action"] and res.get_search_len() == rec[s]["search_len"]
        mz_tree.batch_backpropagate(s + 1, 0.997, rec[s]["reward"], rec[s]["value"], rec[s]["policy"], mm, res, vtp)
    assert roots.get_distributions() == exp["distributions"]
    assert np.array_equal(np.asarray(roots.get_values(), np.float32).view(np.uint32),
                          np.asarray(exp["values"], np.float32).view(np.uint32))


def test_full_size_properties():
    """BASELINE north-star size (1024 roots, 50 simulations, A=18): size-independent invariants."""
    B, A, S = 1024, 18, 50
    ref, cu, obs, mask, legal, noises, mcts = _setup(B, A, S, seed=9, masks=True)
    out = cu.initial_inference(obs.cuda())
    roots = mcts.roots(B, legal)
    roots.prepare(0.25, noises, [0.] * B, out.policy_logits, [-1] * B)
    mcts.search(roots, cu, out.latent_state, [-1] * B)
    v, n = roots.get_distributions_tensor()
    v, n = v.cpu().numpy(), n.cpu().numpy()
    assert (n == mask.sum(1)).all()
    for b in range(B):
        assert (v[b, :n[b]] >= 0).all() and v[b, :n[b]].sum() == S and (v[b, n[b]:] == -1).all()
    vals = np.asarray(roots.get_values())
    assert np.isfinite(vals).all()
    traj = roots.get_trajectories()
    assert all(1 <= len(t) <= S for t in traj)
    # idempotence: same inputs -> same search
    roots2 = mcts.roots(B, legal)
    roots2.prepare(0.25, noises, [0.] * B, out.policy_logits, [-1] * B)
    mcts.search(roots2, cu, out.latent_state, [-1] * B)
    assert np.array_equal(roots2.get_distributions_tensor()[0].cpu().numpy(), v)


def test_collect_policy_matches_manual_composition():
    """lz_search_collect (initial_inference -> reset(mask) -> prepare(noise) -> graph) through the
    _forward_collect mirror, from HOST buffers, equals the step-by-step composition of the public pieces."""
    from lightzero_b200.collect import MuZeroCollectPolicy
    B, A, S = 40, 18, 30
    ref, cu, obs, mask, legal, noises, mcts = _setup(B, A, S, seed=11, masks=True)
    nz = np.zeros((B, A), np.float32)
    for b, n in enumerate(noises):
        nz[b, :len(n)] = n
    pol = MuZeroCollectPolicy(cu, dict(num_simulations=S, deterministic=True, discount_factor=0.997))
    r = pol.search_batch(obs.pin_memory(), mask, nz, None)
    out = cu.initial_inference(obs.cuda(), return_scalar_value=True)
    roots = mcts.roots(B, legal)
    roots.prepare(0.25, noises, [0.] * B, out.policy_logits, [-1] * B)
    mcts.search(roots, cu, out.latent_state, [-1] * B)
    dist = roots.get_distributions()
    for b in range(B):
        assert r["visits"][b, :r["nlegal"][b]].tolist() == dist[b]
    assert np.array_equal(r["values"].numpy().view(np.uint32), np.asarray(roots.get_values(), np.float32).view(np.uint32))
    assert torch.equal(r["policy_logits"], out.policy_logits.cpu())
    assert torch.equal(r["pred_value"], out.value_scalar.cpu())


def test_forward_collect_output_format():
    """policy/muzero.py:801-808: per-env dict keys and types; actions are legal; eval is arg-max."""
    from lightzero_b200.collect import MuZeroCollectPolicy
    B, A, S = 10, 6, 12
    ref, cu, obs, mask, legal, noises, mcts = _setup(B, A, S, seed=13, masks=True)
    pol = MuZeroCollectPolicy(cu, dict(num_simulations=S, deterministic=True, discount_factor=0.997))
    np.random.seed(0)
    out = pol.forward_collect(obs, mask, temperature=1.0, to_play=[-1])
    assert sorted(out.keys()) == list(range(B))
    for i in range(B):
        o = out[i]
        assert set(o) == {'action', 'visit_count_distributions', 'visit_count_distribution_entropy',
                          'searched_value', 'predicted_value', 'predicted_policy_logits'}
        assert mask[i, o['action']] == 1 and sum(o['visit_count_distributions']) == S
        assert len(o['visit_count_distributions']) == int(mask[i].sum()) and len(o['predicted_policy_logits']) == A
    ev = pol.forward_eval(obs, mask, to_play=[-1])
    for i in range(B):
        d = ev[i]['visit_count_distributions']
        assert ev[i]['action'] == np.nonzero(mask[i])[0][int(np.argmax(d))]


def test_config3_shard_200_simulations():
    """BASELINE config 3 per-GPU shard: 1024 roots over 8 GPUs = 128 roots, num_simulations=200 (deep trees, 201 latent
    slots): persistent search == step-wise drive, bit for bit."""
    B, A, S = 128, 18, 200
    ref, cu, obs, mask, legal, noises, mcts = _setup(B, A, S, seed=21, masks=True, math="tc3")
    out = cu.initial_inference(obs.cuda())
    res = []
    for mode in ("fused", "step"):
        roots = mcts.roots(B, legal)
        roots.prepare(0.25, noises, [0.] * B, out.policy_logits, [-1] * B)
        mcts.search(roots, cu if mode == "fused" else _Recorder(cu), out.latent_state, [-1] * B)
        res.append((roots.get_distributions(), np.asarray(roots.get_values(), np.float32).view(np.uint32).tolist(),
                    roots.get_trajectories()))
        roots.clear()
    assert res[0] == res[1]
    assert all(sum(d) == S for d in res[0][0])


def test_forward_collect_with_device_side_action_selection():
    """SURVEY 8(f-3): the collector's select_action on the GPU.  Same visit counts as the host path; every chosen action is a
    legal, visited one; the entropy equals the host formula."""
    from lightzero_b200.collect import MuZeroCollectPolicy, select_action
    B, A, S = 24, 18, 20
    ref, cu, obs, mask, legal, noises, mcts = _setup(B, A, S, seed=13, masks=True)
    pol = MuZeroCollectPolicy(cu, dict(num_simulations=S, deterministic=True, discount_factor=0.997))
    np.random.seed(0)
    host = pol.forward_collect(obs, mask, temperature=0.5, to_play=[-1])
    np.random.seed(0)
    dev = pol.forward_collect(obs, mask, temperature=0.5, to_play=[-1], device_select_action=True, seed=7)
    for i in range(B):
        assert dev[i]["visit_count_distributions"] == host[i]["visit_count_distributions"]
        a = dev[i]["action"]
        assert mask[i, a] == 1 and dev[i]["visit_count_distributions"][legal[i].index(a)] > 0
        _, e = select_action(np.asarray(dev[i]["visit_count_distributions"]), temperature=0.5, deterministic=True)
        assert abs(dev[i]["visit_count_distribution_entropy"] - e) < 1e-5


def test_fused_search_with_reuse_equals_stepwise_drive():
    """MuZeroMCTSCtree.search_with_reuse (mcts_ctree.py:370-468) as one CUDA graph vs the reference's driver loop restated over
    the mirror's batch_traverse_with_reuse / batch_backpropagate_with_reuse and the same CUDA model (compacted inference
    batch, no_inference_lst / reuse_lst built as the driver does): identical visit counts, value bits and inference counts."""
    from lightzero_b200 import mz_tree
    B, A, S = 96, 6, 30
    ref, cu, obs, mask, legal, noises, mcts = _setup(B, A, S, seed=21, masks=True)
    out = cu.initial_inference(obs.cuda())
    rng = np.random.default_rng(3)
    true_action = [int(l[rng.integers(len(l))]) for l in legal]
    reuse_value = (rng.standard_normal(B) * 0.5).astype(np.float32).tolist()
    roots = mcts.roots(B, legal)
    roots.prepare(0.25, noises, [0.] * B, out.policy_logits, [-1] * B)
    length, avg = mcts.search_with_reuse(roots, cu, out.latent_state, [-1] * B, true_action, reuse_value)
    fused = (roots.get_distributions(), np.asarray(roots.get_values(), np.float32).view(np.uint32).tolist())
    roots.clear()
    # step-wise: the reference loop
    mz_tree.DEFAULT_MAX_SIMS = max(mz_tree.DEFAULT_MAX_SIMS, S)
    roots = mz_tree.Roots(B, legal)
    roots.prepare(0.25, noises, [0.] * B, out.policy_logits, [-1] * B)
    mm = mz_tree.MinMaxStatsList(B)
    mm.set_delta(0.01)
    pool, counts = [out.latent_state], []
    for s in range(S):
        res = mz_tree.ResultsWrapper(B)
        ix, iy, la, vtp = mz_tree.batch_traverse_with_reuse(roots, 19652, 1.25, 0.997, mm, res, [-1] * B, true_action, reuse_value)
        lat, acts, no_inf, reuse = [], [], [], []
        for count, (x, y) in enumerate(zip(ix, iy)):
            if x != -1:
                lat.append(pool[x][y]); acts.append(la[count])
            else:
                no_inf.append(y)
            if x == 0 and la[count] == true_action[count]:
                reuse.append(count)
        counts.append(len(acts))
        if acts:
            o = cu.recurrent_inference(torch.stack(lat), torch.tensor(acts), return_scalars=True)
            pool.append(o.latent_state)
            r, v, p = o.reward_scalar, o.value_scalar, o.policy_logits
        else:
            pool.append([]); r, v, p = [], [], []
        no_inf.append(-1); reuse.append(-1)
        mz_tree.batch_backpropagate_with_reuse(s + 1, 0.997, r, v, p, mm, res, vtp, no_inf, reuse, reuse_value)
    step = (roots.get_distributions(), np.asarray(roots.get_values(), np.float32).view(np.uint32).tolist())
    assert fused == step
    assert length == counts[-1] and abs(avg - sum(counts) / S) < 1e-9
    assert min(counts) < B       # some trees reused a value instead of calling the network
    assert mcts.last_num_kernels == 1 + 2 * S     # traverse + S x (network, back-up(+traverse))


def test_uint8_frames_equal_scaled_float_frames_bit_for_bit():
    """lz_search_collect*_u8: uint8 frames scaled inside the first conv kernel == the float frames the reference's env wrapper
    produces ((obs - 0) / 255 in float64, cast to float32: ScaledFloatFrameWrapper, zoo/atari/envs/atari_wrappers.py:219-220),
    through the host entry point and the device entry point."""
    from lightzero_b200.collect import MuZeroCollectPolicy
    B, A, S = 48, 6, 12
    ref, cu, obs, mask, legal, noises, mcts = _setup(B, A, S, seed=5, math="tc3")
    g = torch.Generator().manual_seed(3)
    u8 = torch.randint(0, 256, (B, 4, 84, 84), dtype=torch.uint8, generator=g)
    f32 = torch.from_numpy((u8.numpy() / 255.).astype(np.float32))
    pol = MuZeroCollectPolicy(cu, dict(num_simulations=S, deterministic=True, discount_factor=0.997))
    noise = np.zeros((B, A), np.float32)
    for b in range(B):
        noise[b, :len(noises[b])] = noises[b]
    res = []
    for o in (f32.pin_memory(), u8.pin_memory(), u8.cuda(), f32.cuda()):
        r = pol.search_batch(o, torch.from_numpy(mask), torch.from_numpy(noise), None, deterministic=True, read_back=True)
        res.append({k: v.clone() for k, v in r.items()})
    for r in res[1:]:
        for k in ("visits", "values", "pred_value", "policy_logits"):
            assert torch.equal(res[0][k].view(torch.int32) if res[0][k].dtype == torch.float32 else res[0][k],
                               r[k].view(torch.int32) if r[k].dtype == torch.float32 else r[k]), k


def test_weight_reload_and_parameter_change_recapture_the_search_graph():
    """A captured search graph bakes in device pointers of the model tables and the tree parameters (by value): reloading the
    weights (the collector's weight sync) or changing discount / value_delta_max must not replay a stale graph."""
    import lightzero_b200 as lzb
    from oracle.model_ref import MuZeroModelRef, emulate_trained_
    B, A, S = 40, 6, 16
    ref, cu, obs, mask, legal, noises, mcts = _setup(B, A, S, seed=3, math="tc3")
    ref2 = emulate_trained_(MuZeroModelRef((4, 84, 84), A), 77)

    def run(model, m):
        out = model.initial_inference(obs.cuda())
        roots = m.roots(B, legal)
        roots.prepare(0.25, noises, [0.] * B, out.policy_logits, [-1] * B)
        m.search(roots, model, out.latent_state, [-1] * B)
        r = (roots.get_distributions(), np.asarray(roots.get_values(), np.float32).view(np.uint32).tolist())
        roots.clear()
        return r

    first = run(cu, mcts)
    cu.load_state_dict(ref2.state_dict())                       # same lz_model, new device tables
    reloaded = run(cu, mcts)
    fresh = lzb.MuZeroModel(observation_shape=(4, 84, 84), action_space_size=A).load_state_dict(ref2.state_dict())
    assert reloaded == run(fresh, mcts) and reloaded != first
    # tree parameters: the fused graph must follow the step-wise drive after a discount change on the same pooled tree
    mcts2 = lzb.MuZeroMCTSCtree(dict(num_simulations=S, deterministic=True, discount_factor=0.9, value_delta_max=0.05))
    fused = run(cu, mcts2)
    step = run_step = None
    out = cu.initial_inference(obs.cuda())
    roots = mcts2.roots(B, legal)
    roots.prepare(0.25, noises, [0.] * B, out.policy_logits, [-1] * B)
    mcts2.search(roots, _Recorder(cu), out.latent_state, [-1] * B)
    step = (roots.get_distributions(), np.asarray(roots.get_values(), np.float32).view(np.uint32).tolist())
    roots.clear()
    assert fused == step and fused != reloaded


class _ToyWorldModel:
    """A deterministic stand-in with the UniZero world model's search-time signature (mcts_ctree.py:160-176): CPU fp32 torch, so
    the reference-side loop and the CUDA-tree driver see identical numbers as long as the trees agree."""

    def __init__(self, A, D=24, K=601, seed=0):
        g = torch.Generator().manual_seed(seed)
        self.A, self.D, self.K = A, D, K
        self.W1 = torch.randn(D, D, generator=g) * 0.4
        self.W2 = torch.randn(A, D, generator=g)
        self.Wv = torch.randn(D, K, generator=g) * 0.5
        self.Wr = torch.randn(D, K, generator=g) * 0.5
        self.Wp = torch.randn(D, A, generator=g)
        self.calls = []

    def recurrent_inference(self, state_action_history, simulation_index, search_depth, timestep=None, task_id=None):
        from lightzero_b200.muzero_model import MZNetworkOutput
        assert len(state_action_history) == simulation_index + 1 and len(search_depth) == state_action_history[-1][0].shape[0]
        lat, act = state_action_history[-1]
        self.calls.append((simulation_index, list(search_depth), timestep))
        x = torch.from_numpy(np.asarray(lat, np.float32))
        a = torch.nn.functional.one_hot(act.cpu().long(), self.A).float()
        nl = torch.tanh(x @ self.W1 + a @ self.W2)
        # fully peaked categorical outputs: softmax . support is then EXACTLY one support value in any correct fp32 softmax, so the
        # 1e-7-level differences between softmax implementations cannot flip a PUCT arg-max and the comparison can be bit for bit
        peak = lambda z: 200.0 * torch.nn.functional.one_hot(z.argmax(1) % 41 + 280, self.K).float()
        return MZNetworkOutput(peak(nl @ self.Wv), peak(nl @ self.Wr), nl @ self.Wp, nl)


@pytest.mark.parametrize("timestep", [None, 7])
def test_unizero_driver_matches_reference_loop(timestep):
    """UniZeroMCTSCtree (mcts_ctree.py:19-208) on the CUDA trees vs the restated reference loop on the compiled reference
    mz_tree, same toy world model: first_action_latent_map, visit counts and root-value bits."""
    import lightzero_b200 as lzb
    from oracle.search_ref import SearchRef, load_tree_module, unizero_search_ref
    B, A, S, D = 40, 9, 30, 24
    rng = np.random.default_rng(3)
    mask = (rng.random((B, A)) < 0.7).astype(np.uint8)
    mask[np.arange(B), rng.integers(0, A, B)] = 1
    legal = [np.nonzero(mask[b])[0].tolist() for b in range(B)]
    noises = [rng.dirichlet([0.3] * len(l)).astype(np.float32).tolist() for l in legal]
    lat0 = rng.standard_normal((B, D)).astype(np.float32)
    logits0 = rng.standard_normal((B, A)).astype(np.float32)
    tree, kind = load_tree_module()
    sref = SearchRef(tree, num_simulations=S, deterministic=True)
    r_ref = sref.roots(B, legal, action_space_size=A)
    r_ref.prepare(0.25, noises, [0.] * B, logits0.tolist(), [-1] * B)
    m_ref = _ToyWorldModel(A, D)
    map_ref = unizero_search_ref(sref, r_ref, m_ref, lat0, [-1] * B, timestep=timestep)

    mcts = lzb.UniZeroMCTSCtree(dict(num_simulations=S, deterministic=True, discount_factor=0.997, device="cpu"))
    roots = mcts.roots(B, legal)
    roots.prepare(0.25, noises, [0.] * B, logits0.tolist(), [-1] * B)
    m_cu = _ToyWorldModel(A, D)
    map_cu = mcts.search(roots, m_cu, lat0, [-1] * B, timestep=timestep)
    assert m_cu.calls == m_ref.calls
    assert roots.get_distributions() == r_ref.get_distributions()
    assert np.array_equal(np.asarray(roots.get_values(), np.float32).view(np.uint32),
                          np.asarray(r_ref.get_values(), np.float32).view(np.uint32))
    assert [sorted(m.keys()) for m in map_cu.values()] == [sorted(m.keys()) for m in map_ref.values()]
    for e in range(B):
        for a, v in map_ref[e].items():
            assert np.array_equal(np.asarray(map_cu[e][a]), np.asarray(v))
