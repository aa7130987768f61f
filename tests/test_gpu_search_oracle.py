"""The fused searches against the C oracle driving the same network, bit for bit.

The oracle (oracle/ctree_port.c, pinned to the compiled reference) picks every leaf; the CUDA network evaluates it:
per simulation the latents are gathered from a pool at the oracle's (ix, iy), ``recurrent_inference(...,
return_scalars=True)`` runs them, and the kernel's own scalars and logits go into the oracle's back-up.  The fused
``MuZeroMCTSCtree.search`` on the same roots, noise and to_play must then give the same visit counts, root-value bits
and trajectories.  This holds because k_net_tc's per-root outputs do not depend on the root's slot or CTA packing
(test_gpu_net_layers.py) and the persistent search backs up the joint read-out scalars that return_scalars returns
(the same epilogue writes both).  Stochastic cases run the oracle in hash mode with the epoch the device used
(lz_tree_debug_rng) and steps 0 ... S-1, the steps a fused search takes.

Every case asserts that it reached the branch it is named for, from the oracle's tie statistics and the launch plan
(lz_search_debug_plan), and prints them.
"""
import time

import numpy as np
import pytest
import torch

from test_gpu_net_layers import make_latents, make_models

pytestmark = pytest.mark.gpu

SUPPORT_SMALL = (-10., 11., 1.)


# ------------------------------------------------------------------------------------------------ model mutations
def _last_linear(module):
    return [m for m in module.modules() if isinstance(m, torch.nn.Linear)][-1]


@torch.no_grad()
def zero_policy(ref):
    """policy FC2 weights and bias zero: every prior is uniform, unvisited siblings tie exactly"""
    fc = _last_linear(ref.prediction_network.fc_policy)
    fc.weight.zero_()
    fc.bias.zero_()


@torch.no_grad()
def near_policy(ref):
    """policy logits = FC2 bias only, 3e-7 apart (decreasing, so the later children fall into the tie list of the first):
    tie lists with unequal scores within the 1e-6 epsilon"""
    fc = _last_linear(ref.prediction_network.fc_policy)
    fc.weight.zero_()
    fc.bias.copy_(-3e-7 * torch.arange(fc.bias.numel(), dtype=fc.bias.dtype))


@torch.no_grad()
def peaked_zero_values(ref):
    """A = 2 with prior odds e^5 : 1, and value = reward = 0 (all mass on support 0): PUCT follows the likely action, so the
    search path grows by about one level per simulation"""
    fc = _last_linear(ref.prediction_network.fc_policy)
    fc.weight.zero_()
    fc.bias.copy_(torch.tensor([2.5, -2.5]))
    for head in (ref.prediction_network.fc_value, ref.dynamics_network.fc_reward_head):
        fc = _last_linear(head)
        fc.weight.zero_()
        fc.bias.fill_(-1000.0)
        fc.bias[fc.bias.numel() // 2] = 0.0


# ------------------------------------------------------------------------------------------------ the two searches
def _inputs(B, A, seed, players, masks=True, noise=True, tie_root=False):
    rng = np.random.default_rng(seed)
    legal = []
    for b in range(B):
        m = (rng.random(A) < 0.6) if masks else np.ones(A, bool)
        if not m.any():
            m[rng.integers(A)] = True
        legal.append(np.nonzero(m)[0].tolist())
    if masks and A > 1:
        legal[0] = [A - 1]                      # a root with a single legal action (not a prefix)
        legal[-1] = sorted({A - 1, A // 2})     # a root with fewer legal actions than interior nodes have
    logits = np.zeros((B, A), np.float32) if tie_root else (rng.integers(-2, 3, (B, A)) * 0.5).astype(np.float32)
    noises = [rng.dirichlet([0.3] * len(l)).astype(np.float32).tolist() for l in legal] if noise else None
    if players == "1p":
        tp = [-1] * B
    elif players == "2p":
        tp = rng.integers(1, 3, B).tolist()
    else:
        tp = rng.choice([-1, 1, 2], B).tolist()
        tp[0], tp[-1] = -1, 1
    return legal, logits, noises, tp


def _prepare(roots, logits, noises, tp):
    B = len(tp)
    if noises is None:
        roots.prepare_no_noise([0.] * B, logits, tp)
    else:
        roots.prepare(0.25, noises, [0.] * B, logits, tp)


def debug_rng(roots):
    from lightzero_b200 import cabi
    t = roots._tree
    key = np.zeros(2, np.uint64)
    step = np.zeros(1, np.uint32)
    cabi.check(t.lib.lz_tree_debug_rng(t.h, key.ctypes.data, key[1:].ctypes.data, step.ctypes.data), "lz_tree_debug_rng")
    return int(key[0]), int(key[1]), int(step[0])


def debug_plan(roots, model, S):
    from lightzero_b200 import cabi
    t = roots._tree
    info = np.zeros(8, np.int32)
    cabi.check(t.lib.lz_search_debug_plan(t.search_for(model, S), info.ctypes.data), "lz_search_debug_plan")
    return dict(zip(("persistent", "R", "ctas", "last", "pbc_smem", "b2_smem", "layers", "N"), (int(v) for v in info)))


def fused_search(cu, mcts, S, latent, legal, logits, noises, tp, cap=None, roots=None):
    """MuZeroMCTSCtree.search; `cap`: tree capacity (max_sims) larger than S"""
    if roots is None:
        roots = mcts.roots(len(tp), legal)
    _prepare(roots, logits, noises, tp)
    if cap is not None:
        roots._materialize(cap)
    mcts.search(roots, cu, latent, tp)
    res = (roots.get_distributions(), np.asarray(roots.get_values(), np.float32).view(np.uint32).tolist(),
           roots.get_trajectories())
    return res, debug_rng(roots), debug_plan(roots, cu, S), roots


def oracle_search(cu, S, latent, legal, logits, noises, tp, det, key=None, step0=0, variant=0, discount=0.997, delta=0.01):
    """The reference loop (mcts_ctree.py:281-368) on the C oracle, with the CUDA network evaluating the leaves"""
    from oracle import ctree_port as port
    B, A = len(tp), logits.shape[1]
    roots = port.Roots(B, legal, action_space_size=A, max_sims=S)
    _prepare(roots, logits.tolist(), noises, tp)
    if not det:
        roots.set_tie_hash(key[0], key[1], step0, variant)
    mm = port.MinMaxStatsList(B)
    mm.set_delta(delta)
    pool = torch.empty((S + 1,) + tuple(latent.shape), device="cuda")
    pool[0] = latent
    with torch.no_grad():
        for s in range(S):
            res = port.ResultsWrapper(B)
            ix, iy, la, vtp = port.batch_traverse(roots, 19652, 1.25, discount, mm, res, list(tp), det)
            o = cu.recurrent_inference(pool[torch.tensor(ix, device="cuda"), torch.tensor(iy, device="cuda")],
                                       torch.tensor(la, device="cuda"), return_scalars=True)
            pool[s + 1] = o.latent_state
            port.batch_backpropagate(s + 1, discount, o.reward_scalar.cpu().numpy(), o.value_scalar.cpu().numpy(),
                                     o.policy_logits.cpu().numpy(), mm, res, vtp)
    out = (roots.get_distributions(), np.asarray(roots.get_values(), np.float32).view(np.uint32).tolist(),
           roots.get_trajectories())
    return out, roots.tie_stats()


def _report(name, st, plan, players, kernels, seconds):
    stage = "none" if not plan["persistent"] else f"pbc:{'smem' if plan['pbc_smem'] else 'global'}/b2:{'smem' if plan['b2_smem'] else 'global'}"
    print(f"\n[search-oracle] {name}: ties={st['ties']} draws={st['draws']} near={st['near']} max_len={st['max_len']} "
          f"players={players} R={plan['R']} ctas={plan['ctas']} last={plan['last']} layers={plan['layers']} N={plan['N']} "
          f"staging={stage} kernels={kernels} {seconds:.1f}s")


# ------------------------------------------------------------------------------------------------ the case matrix
# name: A, B, S, deterministic, players, model kwargs, input kwargs, tree capacity, expected staging (pbc, b2) or None
CASES = {
    "a6_b131_det_1p": (6, 131, 50, True, "1p", {}, {}, None, (1, 1)),
    "a6_b131_sto_1p": (6, 131, 50, False, "1p", {}, {}, None, (1, 1)),
    "a18_b1201_sto_2p": (18, 1201, 30, False, "2p", {}, {}, None, (1, 1)),
    "a6_b7_sto_mixed": (6, 7, 50, False, "mixed", {}, {}, None, (1, 1)),
    "a2_b7_s200_sto_peaked": (2, 7, 200, False, "1p", dict(mutate=peaked_zero_values), dict(noise=False), None, (1, 1)),
    "a1_b3_s200_sto": (1, 3, 200, False, "1p", {}, dict(masks=False), None, (1, 1)),
    "a31_b300_sto_zero_policy": (31, 300, 40, False, "1p", dict(mutate=zero_policy), dict(noise=False, tie_root=True), None, (1, 1)),
    "a32_b531_sto_2p_near_ties": (32, 531, 30, False, "2p", dict(mutate=near_policy), dict(noise=False), None, (1, 1)),
    "a32_b531_det_zero_policy": (32, 531, 30, True, "mixed", dict(mutate=zero_policy), dict(noise=False, tie_root=True), None, (1, 1)),
    "a6_b1_s1_sto": (6, 1, 1, False, "1p", {}, dict(noise=False, tie_root=True), None, (1, 1)),
    "a6_b1_s1_det_2p": (6, 1, 1, True, "2p", {}, {}, None, (1, 1)),
    "a6_b64_sto_cap400": (6, 64, 50, False, "2p", {}, {}, 400, (1, 0)),
    "a6_b16_s800_sto": (6, 16, 800, False, "1p", {}, {}, None, (1, 0)),
    "nres3_k21_a9_b5_s600_sto": (9, 5, 600, False, "2p", dict(nres=3, support=SUPPORT_SMALL), {}, None, (0, 1)),
    "nres4_a6_b140_sto_mixed": (6, 140, 40, False, "mixed", dict(nres=4), dict(noise=False, tie_root=True), None, (0, 0)),
    "a33_b40_sto_2p": (33, 40, 20, False, "2p", {}, {}, None, None),
    "tc1_a40_b64_sto": (40, 64, 20, False, "1p", dict(math="tc1"), {}, None, None),
}


@pytest.mark.parametrize("name", list(CASES))
def test_fused_search_equals_oracle_driving_the_same_network(name):
    import lightzero_b200 as lzb
    A, B, S, det, players, mkw, ikw, cap, staging = CASES[name]
    t0 = time.time()
    seed = sum(map(ord, name))
    _, cu = make_models(A=A, seed=seed % 97, **mkw)
    latent = make_latents(B, seed)
    legal, logits, noises, tp = _inputs(B, A, seed, players, **ikw)
    mcts = lzb.MuZeroMCTSCtree(dict(num_simulations=S, deterministic=det, discount_factor=0.997))
    got, key, plan, roots = fused_search(cu, mcts, S, latent, legal, logits, noises, tp, cap=cap)
    exp, st = oracle_search(cu, S, latent, legal, logits, noises, tp, det, key=key)
    kernels = mcts.last_num_kernels
    roots.clear()
    _report(name, st, plan, players, kernels, time.time() - t0)
    assert got[0] == exp[0], "visit counts"
    assert got[1] == exp[1], "root value bits"
    assert got[2] == exp[2], "trajectories"
    assert all(sum(d) == S for d in got[0])
    # the branch the case is named for
    assert plan["N"] == (cap or S) + 1
    if staging is None:
        assert not plan["persistent"] and kernels == 2 * S + 1
    else:
        assert plan["persistent"] and kernels == 1
        assert (plan["pbc_smem"], plan["b2_smem"]) == staging
        R = min(max(-(-B // 132), 1), 8)
        assert plan["R"] == R and plan["ctas"] == -(-B // R) and plan["last"] == B - (plan["ctas"] - 1) * R
    if not det and S > 1 and A > 1:
        assert st["ties"] > 0 and st["draws"] > 0
    if "near" in name:
        assert st["near"] > 0
    if "zero_policy" in name:
        assert st["ties"] >= B * S // 4
    if name.startswith("a1_"):
        assert st["max_len"] == S          # path length == simulation index + 1
    if "peaked" in name:
        assert st["max_len"] >= 64
    if S == 1:
        assert st["max_len"] == 1


def test_mlp_model_multi_kernel_search_equals_oracle():
    """MuZeroModelMLP (vector latents, the multi-kernel search graph), stochastic, two players"""
    import lightzero_b200 as lzb
    from oracle.model_ref import MuZeroModelMLPRef, emulate_trained_mlp_
    A, B, S = 4, 96, 25
    ref = emulate_trained_mlp_(MuZeroModelMLPRef(8, A, res_connection_in_dynamics=True), 3)
    cu = lzb.MuZeroModelMLP(observation_shape=8, action_space_size=A, res_connection_in_dynamics=True).load_state_dict(ref.state_dict())
    g = torch.Generator().manual_seed(4)
    latent = cu.initial_inference(torch.randn(B, 8, generator=g).cuda()).latent_state
    legal, logits, noises, tp = _inputs(B, A, 5, "2p")
    mcts = lzb.MuZeroMCTSCtree(dict(num_simulations=S, deterministic=False, discount_factor=0.997))
    got, key, plan, roots = fused_search(cu, mcts, S, latent, legal, logits, noises, tp)
    exp, st = oracle_search(cu, S, latent, legal, logits, noises, tp, False, key=key)
    kernels = mcts.last_num_kernels
    roots.clear()
    _report("mlp_a4_b96_sto_2p", st, plan, "2p", kernels, 0.0)
    assert got == exp
    assert not plan["persistent"] and kernels == 2 * S + 1 and st["draws"] > 0


def test_discount_and_value_delta_max():
    """non-default discount and MinMax value_delta_max in the persistent kernel"""
    import lightzero_b200 as lzb
    A, B, S = 9, 96, 40
    _, cu = make_models(A=A, seed=31)
    latent = make_latents(B, 31)
    legal, logits, noises, tp = _inputs(B, A, 31, "2p")
    mcts = lzb.MuZeroMCTSCtree(dict(num_simulations=S, deterministic=False, discount_factor=0.9, value_delta_max=0.05))
    got, key, plan, roots = fused_search(cu, mcts, S, latent, legal, logits, noises, tp)
    exp, st = oracle_search(cu, S, latent, legal, logits, noises, tp, False, key=key, discount=0.9, delta=0.05)
    default, _ = oracle_search(cu, S, latent, legal, logits, noises, tp, False, key=key)
    roots.clear()
    _report("a9_b96_sto_2p_discount0.9_delta0.05", st, plan, "2p", mcts.last_num_kernels, 0.0)
    assert got == exp and got[0] != default[0]
    assert plan["persistent"] and st["draws"] > 0


def test_repeated_stochastic_searches_on_one_pooled_tree():
    """Two stochastic searches on the same tree: the second runs at the next epoch, must match the oracle there and must
    differ from the first."""
    import lightzero_b200 as lzb
    A, B, S = 18, 200, 30
    _, cu = make_models(A=A, seed=41, mutate=zero_policy)
    latent = make_latents(B, 41)
    legal, logits, noises, tp = _inputs(B, A, 41, "1p", noise=False, tie_root=True)
    mcts = lzb.MuZeroMCTSCtree(dict(num_simulations=S, deterministic=False, discount_factor=0.997))
    roots = mcts.roots(B, legal)
    first, key1, _, roots = fused_search(cu, mcts, S, latent, legal, logits, noises, tp, roots=roots)
    handle = roots._tree
    second, key2, plan, roots = fused_search(cu, mcts, S, latent, legal, logits, noises, tp, roots=roots)
    assert roots._tree is handle and key2[0] == key1[0] and key2[1] > key1[1]     # every reset advances the epoch
    roots.clear()
    for got, key in ((first, key1), (second, key2)):
        exp, st = oracle_search(cu, S, latent, legal, logits, noises, tp, False, key=key)
        assert got == exp
    _report("a18_b200_sto_repeated", st, plan, "1p", mcts.last_num_kernels, 0.0)
    assert first[0] != second[0]


def test_sensitivity_of_the_stochastic_comparison():
    """Oracle mutations the comparison must catch on tie-rich roots (the device is unchanged): the wrong epoch, the wrong
    step, the tie after the drawn one, and the deterministic rule.  Each must disagree with the device on most roots."""
    import lightzero_b200 as lzb
    A, B, S = 31, 132, 30
    _, cu = make_models(A=A, seed=51, mutate=zero_policy)
    latent = make_latents(B, 51)
    legal, logits, noises, tp = _inputs(B, A, 51, "1p", noise=False, tie_root=True)
    mcts = lzb.MuZeroMCTSCtree(dict(num_simulations=S, deterministic=False, discount_factor=0.997))
    got, key, plan, roots = fused_search(cu, mcts, S, latent, legal, logits, noises, tp)
    roots.clear()
    exp, _ = oracle_search(cu, S, latent, legal, logits, noises, tp, False, key=key)
    assert got == exp

    def frac(o):
        return np.mean([g != e or gv != ev for g, e, gv, ev in zip(got[0], o[0], got[1], o[1])])
    fr = {
        "epoch+1": frac(oracle_search(cu, S, latent, legal, logits, noises, tp, False, key=(key[0], key[1] + 1))[0]),
        "step+1": frac(oracle_search(cu, S, latent, legal, logits, noises, tp, False, key=key, step0=1)[0]),
        "ties[(r+1)%n]": frac(oracle_search(cu, S, latent, legal, logits, noises, tp, False, key=key, variant=2)[0]),
        "deterministic": frac(oracle_search(cu, S, latent, legal, logits, noises, tp, True)[0]),
    }
    print("\n[search-oracle] sensitivity, fraction of roots that disagree: " + ", ".join(f"{k} {v:.3f}" for k, v in fr.items()))
    assert min(fr.values()) > 0.5, fr
