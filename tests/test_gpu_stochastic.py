"""GPU tests of Stochastic MuZero on vector observations (StochasticMuZeroModelMLP, stochastic device trees,
StochasticMuZeroMCTSCtree):
- the model: initial_inference and both recurrent programs against the reference class's fixtures and the float64
  restatement (1e-5 on latents and logits, 2e-4 on scalars) at batches with a partial last CTA and a second wave; a masked
  launch computes the selected rows bit for bit as an unmasked one and leaves every other row untouched;
- the trees: with the chance draw pinned (chance_seed), the device trees driven step by step by the reference's own search
  loop, and the fused search, equal the compiled reference tree (random_device and rand() pinned) driving the same network,
  bit for bit: visit counts, root-value bits, trajectories;
- sampling (chance_seed=None): the outcome frequencies of 2^17 root draws match the priors within 5 binomial sigmas, the whole
  sampled search repeats bit for bit for a fixed RNG key, and the draws of one descent are keyed by depth;
- the fused search on a side stream next to a busy legacy default stream (tests/test_gpu_streams.py's harness);
- the reuse search is refused on stochastic trees, and only the stochastic model keeps afterstate_* tensors."""
import hashlib
import os

import numpy as np
import pytest
import torch

import stoch_mlp_model_ref as SR
from conftest import ROOT
from test_gpu_streams import _check_on_side_stream, sleep_rate  # noqa: F401  (the streams harness and its fixture)

pytestmark = pytest.mark.gpu

NAMES = list(SR.CONFIGS)
GOLDEN = os.path.join(ROOT, "tests", "golden")


def make(name, seed=0):
    import lightzero_b200 as lzb
    ref = SR.build(name, seed)
    sd = dict(ref.state_dict())
    sd["chance_encoder.encoder.0.weight"] = torch.randn(8, 8)     # training-only keys ride along and are ignored
    return ref, lzb.StochasticMuZeroModelMLP(**SR.model_kwargs(name)).load_state_dict(sd)


def close(got, exp, what, tol=1e-5):
    got, exp = np.asarray(got, np.float64), np.asarray(exp, np.float64)
    err = np.abs(got - exp) - tol * np.abs(exp)
    assert err.max() <= tol, f"{what}: max excess {err.max():.3g}"


def scalar(logits, support):
    x = torch.as_tensor(np.asarray(logits)).double()
    v = (torch.softmax(x, -1) * torch.arange(*support, dtype=torch.float64)).sum(-1)
    eps = 0.001
    return (torch.sign(v) * (((torch.sqrt(1 + 4 * eps * (torch.abs(v) + 1 + eps)) - 1) / (2 * eps)) ** 2 - 1)).numpy()


@pytest.mark.parametrize("name", NAMES)
def test_model_matches_fixture(name):
    ref, cu = make(name, NAMES.index(name))
    z = np.load(os.path.join(GOLDEN, f"stoch_mlp_{name}.npz"))
    h = hashlib.sha256()
    for k, v in sorted(ref.state_dict().items()):
        if v.dtype.is_floating_point:
            h.update(k.encode())
            h.update(v.numpy().tobytes())
    assert str(z["weights_sha256"]) == h.hexdigest()      # the fixture was made from these weights
    obs = torch.from_numpy(z["obs"]).cuda()
    o = cu.initial_inference(obs)
    for f in ("value", "policy_logits", "latent_state"):
        close(getattr(o, f).cpu(), z["init_" + f], f"{name} initial {f}")
    a = cu.recurrent_inference(torch.from_numpy(z["init_latent_state"]).cuda(), torch.from_numpy(z["action"]).cuda(), False)
    r = cu.recurrent_inference(torch.from_numpy(z["after_latent_state"]).cuda(), torch.from_numpy(z["chance"]).cuda(), True)
    for f in ("value", "reward", "policy_logits", "latent_state"):
        close(getattr(a, f).cpu(), z["after_" + f], f"{name} afterstate {f}")
        close(getattr(r, f).cpu(), z["rec_" + f], f"{name} dynamics {f}")


@pytest.mark.parametrize("name", ["cartpole", "lunarlander_disc", "l32_c1_h1", "l256_c608"])
@pytest.mark.parametrize("B", [65, 64 * 132 + 37])
def test_model_float64(name, B):
    seed = NAMES.index(name)
    ref, cu = make(name, seed)
    ref64 = SR.build(name, seed, torch.float64)
    obs_dim, A, C, L, _, _, sup = SR.CONFIGS[name]
    g = torch.Generator().manual_seed(B)
    obs = torch.rand((B, obs_dim), generator=g) * 2 - 1
    act, ch = torch.randint(0, A, (B,), generator=g), torch.randint(0, C, (B,), generator=g)
    o = cu.initial_inference(obs.cuda(), return_scalar_value=True)
    lat = o.latent_state.cpu()
    with torch.no_grad():
        rep = ref64.representation_network      # its forward casts to float32 like the reference's: run its layers in float64
        e_lat = rep.norm(rep.fc_representation(obs.double()))
        e_pol, e_val = ref64.prediction_network(e_lat)
        ea = ref64.recurrent_inference(lat.double(), act, False)
        er = ref64.recurrent_inference(ea.latent_state.float().double(), ch, True)
    close(o.latent_state.cpu(), e_lat, "initial latent")
    close(o.policy_logits.cpu(), e_pol, "initial policy")
    close(o.value_scalar.cpu(), scalar(e_val, sup), "initial value", 2e-4)
    a = cu.recurrent_inference(lat.cuda(), act.cuda(), False, return_scalars=True)
    r = cu.recurrent_inference(ea.latent_state.float().cuda(), ch.cuda(), True, return_scalars=True)
    for got, exp in ((a, ea), (r, er)):
        close(got.latent_state.cpu(), exp.latent_state, "latent")
        close(got.policy_logits.cpu(), exp.policy_logits, "policy")
        close(got.value.cpu(), exp.value, "value logits")
        close(got.reward.cpu(), exp.reward, "reward logits")
        close(got.value_scalar.cpu(), scalar(exp.value, sup), "value", 2e-4)
        close(got.reward_scalar.cpu(), scalar(exp.reward, sup), "reward", 2e-4)


@pytest.mark.parametrize("afterstate", [False, True])
def test_masked_launch(afterstate):
    from lightzero_b200 import cabi
    _, cu = make("l64_c9_res", NAMES.index("l64_c9_res"))
    A, C, L = cu.action_space_size, cu.chance_space_size, cu.latent_state_dim
    B = 200
    g = torch.Generator().manual_seed(3)
    state = torch.randn(B, L, generator=g).cuda()
    opt = torch.randint(0, C if afterstate else A, (B,), generator=g).int().cuda()
    mask = torch.randint(0, 4, (B,), generator=g).int().cuda()
    mask[64:128] = 0       # one CTA with no selected row
    full = cu.recurrent_inference(state, opt, afterstate, return_scalars=True)
    P = A if afterstate else C
    outs = [torch.full(s, 7.25, device="cuda") for s in ((B, L), (B, cu.reward_support_size), (B, cu.value_support_size),
                                                          (B, P), (B,), (B,))]
    lib = cu._lib
    cabi.check(lib.lz_model_recurrent_inference_stochastic(cu._h, int(afterstate), B, state.data_ptr(), opt.data_ptr(),
                                                           mask.data_ptr(), 1, *(o.data_ptr() for o in outs),
                                                           cabi.stream_ptr()), "masked")
    sel = (mask & 1) == 1
    exp = (full.latent_state, full.reward, full.value, full.policy_logits, full.reward_scalar, full.value_scalar)
    for got, e in zip(outs, exp):
        assert torch.equal(got[sel], e[sel])
        assert bool((got[~sel] == 7.25).all())


# ---- trees -------------------------------------------------------------------------------------------------------------
def reference_loop(T, model, lat, legal, logits, noises, to_play, S, chance_seed):
    """mcts_ctree_stochastic.py:117-252 (oracle/tree_drive.py, kind "stoch") with the module T (the compiled reference or
    lightzero_b200.stochastic_mz_tree) driving `model`; the network's own scalars (softmax . support -> h^-1 in the kernel) are
    what both trees back up.  Decision ties take the first maximum.  Returns (the drive's trace, roots)."""
    from oracle.tree_drive import drive, network
    c = dict(B=len(to_play), A=model.action_space_size, C=model.chance_space_size, S=S, legal=legal, root_logits=logits,
             noises=noises, to_play=to_play, chance_seed=chance_seed)
    return drive(T, c, "stoch", network(model, lat, stochastic=True), det=True)


def readout(roots):
    return dict(dist=roots.get_distributions(), values=np.asarray(roots.get_values(), np.float32).view(np.uint32),
                traj=roots.get_trajectories())


def assert_equal(a, b):
    assert a["dist"] == [d[:len(x)] for d, x in zip(b["dist"], a["dist"])] and [len(d) for d in a["dist"]] == \
        [len(d) for d in b["dist"]], (a["dist"][:3], b["dist"][:3])
    assert np.array_equal(a["values"], b["values"])
    assert a["traj"] == b["traj"]


def case(name, B, two_player, masked, noise, seed):
    ref, cu = make(name, NAMES.index(name))
    obs_dim, A, C = SR.CONFIGS[name][:3]
    rng = np.random.default_rng(seed)
    obs = torch.from_numpy(rng.uniform(-1, 1, (B, obs_dim)).astype(np.float32)).cuda()
    o = cu.initial_inference(obs)
    legal = [sorted(rng.choice(A, rng.integers(1, A + 1), replace=False).tolist()) if masked else list(range(A))
             for _ in range(B)]
    noises = [rng.dirichlet([0.3] * len(l)).astype(np.float32).tolist() for l in legal] if noise else None
    to_play = [int(x) for x in rng.integers(1, 3, B)] if two_player else [-1] * B
    return cu, o, legal, noises, to_play, C


CASES = [("cartpole", 64, False, False, True, 0, 25), ("lunarlander_disc", 40, False, True, True, 1, 50),
         ("cartpole", 33, True, True, False, 2, 200), ("l64_c9_res", 20, True, False, True, 3, 60),
         ("pendulum_cont_disc", 16, False, True, False, 4, 200), ("l32_c1_h1", 10, False, False, True, 5, 30)]


@pytest.mark.parametrize("name,B,two_player,masked,noise,seed,S", CASES)
def test_tree_parity(name, B, two_player, masked, noise, seed, S):
    from oracle import build_stoch_ref
    import lightzero_b200 as lzb
    from lightzero_b200 import stochastic_mz_tree as T
    oracle = build_stoch_ref.load()
    if oracle is None:
        pytest.skip("compiled reference Stochastic MuZero tree not built")
    cu, o, legal, noises, to_play, C = case(name, B, two_player, masked, noise, seed)
    logits = o.policy_logits.cpu().tolist()
    chance_seed = 1000 + seed

    def prepare(roots):
        if noise:
            roots.prepare(0.25, noises, [0.] * B, logits, to_play)
        else:
            roots.prepare_no_noise([0.] * B, logits, to_play)
        return roots

    from oracle.tree_drive import assert_same
    want, ref_roots = reference_loop(oracle, cu, o.latent_state, legal, logits, noises, to_play, S, chance_seed)
    got, step_roots = reference_loop(T, cu, o.latent_state, legal, logits, noises, to_play, S, chance_seed)
    assert_same(got, want)                  # per simulation is_chance, ix, iy, last_action, search_len, vtp, then the read-outs
    want = readout(ref_roots)
    assert_equal(readout(step_roots), want)
    step_roots.clear()
    mcts = lzb.StochasticMuZeroMCTSCtree(dict(num_simulations=S, deterministic=True, chance_seed=chance_seed))
    roots = prepare(mcts.roots(B, legal, C))
    mcts.search(roots, cu, o.latent_state, to_play)
    assert_equal(readout(roots), want)
    assert all(sum(d) == S for d in readout(roots)["dist"])


def test_sampling_frequencies():
    """chance_seed=None: every root has one legal action, so the second descent of each tree draws the outcome of the same
    chance node; 2^17 trees give the outcome frequencies"""
    from lightzero_b200 import stochastic_mz_tree as T
    _, cu = make("l64_c9_res", NAMES.index("l64_c9_res"))
    B, C = 1 << 17, cu.chance_space_size
    lat = cu.initial_inference(torch.zeros(1, 5).cuda()).latent_state.repeat(B, 1)
    after = cu.recurrent_inference(lat[:1], torch.zeros(1, dtype=torch.int32).cuda(), False)
    roots = T.Roots(B, [[0]] * B, C)
    roots.prepare_no_noise([0.] * B, torch.zeros(B, cu.action_space_size), [-1] * B)
    mm, res = T.MinMaxStatsList(B), T.ResultsWrapper(B)
    mm.set_delta(0.01)
    T.batch_traverse(roots, 19652, 1.25, 0.997, mm, res, [-1] * B, return_tensors=True)
    T.batch_backpropagate(1, 0.997, torch.zeros(B), torch.zeros(B), after.policy_logits.repeat(B, 1), mm, res, [-1] * B,
                          [True] * B, [])
    res = T.ResultsWrapper(B)
    is_chance, _, _, act, _ = T.batch_traverse(roots, 19652, 1.25, 0.997, mm, res, [-1] * B, return_tensors=True)
    assert not bool(is_chance.any())
    counts = torch.bincount(act.long(), minlength=C).cpu().numpy()
    p = torch.softmax(after.policy_logits[0].double(), -1).cpu().numpy()
    sigma = np.sqrt(B * p * (1 - p))
    assert np.all(np.abs(counts - B * p) <= 5 * sigma + 1), (counts, B * p)


def test_search_on_side_stream(sleep_rate):
    """the fused search, model, roots and search created on a side stream, next to a busy legacy default stream: no call waits
    for the default stream and the outputs equal a default-stream run bit for bit (tests/test_gpu_streams.py's harness)"""
    import lightzero_b200 as lzb
    from test_gpu_streams import _readout
    name, B, S = "cartpole", 96, 25
    obs_dim, A, C = SR.CONFIGS[name][:3]
    sd = SR.build(name, NAMES.index(name)).state_dict()
    rng = np.random.default_rng(7)
    x = torch.from_numpy(rng.uniform(-1, 1, (B, obs_dim)).astype(np.float32)).cuda()
    legal = [list(range(A))] * B
    noises = [rng.dirichlet([0.3] * A).astype(np.float32).tolist() for _ in range(B)]

    def scenario():
        m = lzb.StochasticMuZeroModelMLP(**SR.model_kwargs(name)).load_state_dict(sd)
        o = m.initial_inference(x)
        mcts = lzb.StochasticMuZeroMCTSCtree(dict(num_simulations=S, deterministic=True, chance_seed=11))
        roots = mcts.roots(B, legal, C)
        roots.prepare(0.25, noises, [0.] * B, o.policy_logits, [-1] * B)
        mcts.search(roots, m, o.latent_state, [-1] * B)
        out = _readout(roots, max(A, C), S)
        roots.clear()
        out["_keep"] = (m, mcts)
        return out
    _check_on_side_stream(sleep_rate, "stochastic cartpole", scenario)


def test_sampled_search_repeats():
    """chance_seed=None: on two fresh trees with the same RNG key (seed, epoch), the reference loop driving the device trees
    step by step and the fused search draw the same chance outcomes, so the whole sampled search repeats bit for bit"""
    import lightzero_b200 as lzb
    from lightzero_b200 import cabi, stochastic_mz_tree as T
    name, B, S = "l64_c9_res", 77, 30        # a shape no other test pools: both trees are fresh
    cu, o, legal, noises, to_play, C = case(name, B, False, True, True, 9)
    logits = o.policy_logits.cpu().tolist()
    _, step = reference_loop(T, cu, o.latent_state, legal, logits, noises, to_play, S, None)
    got = readout(step)
    mcts = lzb.StochasticMuZeroMCTSCtree(dict(num_simulations=S, deterministic=True, chance_seed=None))
    fused = mcts.roots(B, legal, C)
    fused.prepare(0.25, noises, [0.] * B, logits, to_play)
    mcts.search(fused, cu, o.latent_state, to_play)
    assert fused._tree is not step._tree
    keys = []
    for r in (step, fused):
        seed, epoch, counter = (cabi.ctypes.c_uint64(), cabi.ctypes.c_uint64(), cabi.ctypes.c_uint32())
        cabi.check(r._tree.lib.lz_tree_debug_rng(r._tree.h, cabi.ctypes.byref(seed), cabi.ctypes.byref(epoch),
                                                 cabi.ctypes.byref(counter)), "lz_tree_debug_rng")
        keys.append((seed.value, epoch.value))
    assert keys[0] == keys[1] and keys[0][1] == 1        # the same seed, and one reset each since creation
    assert_equal(readout(fused), got)
    pinned = lzb.StochasticMuZeroMCTSCtree(dict(num_simulations=S, deterministic=True, chance_seed=12345))
    again = pinned.roots(B, legal, C)
    again.prepare(0.25, noises, [0.] * B, logits, to_play)
    pinned.search(again, cu, o.latent_state, to_play)
    assert readout(again)["traj"] != got["traj"]       # the sampled draws are not the pinned ones


def test_draws_keyed_by_depth():
    """one descent through two chance nodes draws two independent outcomes: with two equally likely outcomes at both, the
    depth-1 and depth-3 draws of the last descent agree for about half of 2^14 trees (a key without the depth would make them
    agree always).  Decision nodes have one action, so every descent goes root -> a0 -> chance -> a0 -> chance."""
    from lightzero_b200 import stochastic_mz_tree as T
    B, S = 1 << 14, 10
    roots = T.Roots(B, [[0]] * B, 2, max_simulations=S + 1)
    roots.prepare_no_noise([0.] * B, torch.zeros(B, 1), [-1] * B)
    mm = T.MinMaxStatsList(B)
    mm.set_delta(0.01)
    zeros, pol = torch.zeros(B), torch.zeros(B, 2)
    for sim in range(S):
        res = T.ResultsWrapper(B)
        T.batch_traverse(roots, 19652, 1.25, 0.997, mm, res, [-1] * B, return_tensors=True)
        T.batch_backpropagate(sim + 1, 0.997, zeros, zeros, pol, mm, res, [-1] * B, [], [])
    T.batch_traverse(roots, 19652, 1.25, 0.997, mm, T.ResultsWrapper(B), [-1] * B, return_tensors=True)
    deep = [t for t in roots.get_trajectories() if len(t) >= 4]
    assert len(deep) > B // 2
    same = sum(t[1] == t[3] for t in deep)
    n = len(deep)
    assert abs(same - n / 2) <= 5 * np.sqrt(n / 4), (same, n)


def test_reuse_refused():
    import lightzero_b200 as lzb
    from lightzero_b200 import cabi
    cu, o, legal, noises, to_play, C = case("cartpole", 8, False, False, False, 3)
    mcts = lzb.StochasticMuZeroMCTSCtree(dict(num_simulations=5, chance_seed=1))
    roots = mcts.roots(8, legal, C)
    roots.prepare_no_noise([0.] * 8, o.policy_logits, to_play)
    mcts.search(roots, cu, o.latent_state, to_play)
    with pytest.raises(NotImplementedError):
        mcts.search_with_reuse(roots, cu, o.latent_state, to_play, [0] * 8, [0.] * 8)
    t = roots._tree
    q = t.search_for(cu, 5)
    ta, rv = torch.zeros(8, dtype=torch.int32, device="cuda"), torch.zeros(8, device="cuda")
    with pytest.raises(cabi.LzError, match="stochastic tree"):
        cabi.check(t.lib.lz_search_run_with_reuse(q, o.latent_state.data_ptr(), None, None, ta.data_ptr(), rv.data_ptr(),
                                                  None, cabi.stream_ptr()), "lz_search_run_with_reuse")


def test_afterstate_keys_only_for_the_stochastic_model():
    """lz_model_set_tensor keeps afterstate_* tensors for a StochasticMuZeroModelMLP only; any other model ignores them (1)"""
    import lightzero_b200 as lzb
    from lightzero_b200 import cabi
    x = torch.zeros(4)
    mz = lzb.MuZeroModelMLP(observation_shape=8, action_space_size=4, latent_state_dim=256)
    st = lzb.StochasticMuZeroModelMLP(observation_shape=8, action_space_size=4, chance_space_size=2, latent_state_dim=256)
    for name in ("afterstate_dynamics_network.fc_dynamics.0.bias", "afterstate_prediction_network.fc_value_head.3.bias"):
        assert cabi.check(mz._lib.lz_model_set_tensor(mz._h, name.encode(), x.data_ptr(), 4)) == 1
        assert cabi.check(st._lib.lz_model_set_tensor(st._h, name.encode(), x.data_ptr(), 4)) == 0
