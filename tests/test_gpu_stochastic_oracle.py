"""The fused Stochastic MuZero search against the C oracle driving the same network, bit for bit.

The oracle (oracle/ctree_port.c in stochastic mode, pinned to the compiled reference tree by tests/test_oracle_pin.py) picks
every leaf; the CUDA StochasticMuZeroModelMLP evaluates it: per simulation the latents are gathered at the oracle's (ix, iy),
chance leaves run ``recurrent_inference(afterstate=False)`` and the others ``afterstate=True``, with ``return_scalars=True``,
and the kernel's own scalars and logits go into the oracle's back-up (oracle/tree_drive.py, kind "stoch").  The fused
``StochasticMuZeroMCTSCtree.search`` on the same roots, noise and to_play must then give the same visit counts, root-value bits
and trajectories.

All four draw modes are covered: ``deterministic`` True / False (decision-node ties: the first maximum, or the hashed draw)
times ``chance_seed`` pinned / None (chance nodes: the reference's std::mt19937 draw, or the counter RNG).  Hash-mode cases
read (seed, epoch) from ``lz_tree_debug_rng`` and use steps 0 ... S-1, the steps a fused search takes.

Every case prints and asserts what it reached: chance draws, hashed tie draws with r > 0, the longest path, and the
(simulation, program, CTA) triples of the masked network launches with no selected row (a 64-row CTA whose rows are all of the
other leaf kind)."""
import time

import numpy as np
import pytest
import torch

import stoch_mlp_model_ref as SR
from oracle.tree_drive import assert_same, drive, network, readout

pytestmark = pytest.mark.gpu

CTA_ROWS = 64           # rows per CTA of the MlpTc kernel
SUPPORT_SMALL = (-10., 11., 1.)
CONFIGS = dict(SR.CONFIGS,
               # decision nodes wider than a warp: A = 40 > 32, C = 5
               a40_c5=(7, 40, 5, 64, True, 16, (-300., 301., 1.)),
               # one action and one outcome: every descent goes one level deeper than the last
               a1_c1=(4, 1, 1, 32, True, 8, SUPPORT_SMALL))


# ------------------------------------------------------------------------------------------------ models
def _last_linear(module):
    return [m for m in module.modules() if isinstance(m, torch.nn.Linear)][-1]


def _policy_heads(ref):
    """the decision policy (prediction) and the chance policy (afterstate prediction)"""
    return [ref.prediction_network.fc_policy_head, ref.afterstate_prediction_network.fc_policy_head]


@torch.no_grad()
def zero_policy(ref):
    """both policy FC2s zero: uniform priors, exact ties between unvisited siblings and uniform chance priors"""
    for head in _policy_heads(ref):
        fc = _last_linear(head)
        fc.weight.zero_()
        fc.bias.zero_()


@torch.no_grad()
def near_policy(ref):
    """both policy heads' logits = FC2 bias only, 3e-7 apart (decreasing): tie lists with unequal scores within 1e-6"""
    for head in _policy_heads(ref):
        fc = _last_linear(head)
        fc.weight.zero_()
        fc.bias.copy_(-3e-7 * torch.arange(fc.bias.numel(), dtype=fc.bias.dtype))


@torch.no_grad()
def large_scalars(ref):
    """value and reward heads peaked on support entries above 10^3 after h^-1: scalars in the thousands"""
    heads = (ref.prediction_network.fc_value_head, ref.afterstate_prediction_network.fc_value_head,
             ref.dynamics_network.fc_reward_head, ref.afterstate_dynamics_network.fc_reward_head)
    for i, head in enumerate(heads):
        fc = _last_linear(head)
        fc.weight.mul_(0.05)
        fc.bias[250 + 13 * i] += 12.0           # support value -50 + 13 i ... and
        fc.bias[540 + 7 * i] += 12.5            # 240 + 7 i: h^-1 gives about 3e3 .. 6e3


_models = {}


def make(name, mutate=None):
    import lightzero_b200 as lzb
    key = (name, mutate.__name__ if mutate else None)
    if key not in _models:
        seed = sorted(CONFIGS).index(name)
        torch.manual_seed(seed)
        from oracle.model_ref import emulate_trained_mlp_
        ref = emulate_trained_mlp_(SR.StochasticMuZeroModelMLPRef(*CONFIGS[name]), seed).eval()
        if mutate is not None:
            mutate(ref)
        obs, A, C, L, res, hid, sup = CONFIGS[name]
        kw = dict(observation_shape=obs, action_space_size=A, chance_space_size=C, latent_state_dim=L,
                  res_connection_in_dynamics=res, reward_head_hidden_channels=[hid], value_head_hidden_channels=[hid],
                  policy_head_hidden_channels=[hid], reward_support_range=sup, value_support_range=sup)
        _models[key] = lzb.StochasticMuZeroModelMLP(**kw).load_state_dict(ref.state_dict())
    return _models[key]


# ------------------------------------------------------------------------------------------------ the two searches
def _inputs(cu, B, seed, players, masks=True, noise=True):
    A = cu.action_space_size
    rng = np.random.default_rng(seed)
    obs = torch.from_numpy(rng.uniform(-1, 1, (B, cu.observation_shape)).astype(np.float32)).cuda()
    o = cu.initial_inference(obs)
    legal = []
    for b in range(B):
        m = (rng.random(A) < 0.6) if masks else np.ones(A, bool)
        if not m.any():
            m[rng.integers(A)] = True
        legal.append(np.nonzero(m)[0].tolist())
    if masks and A > 1:
        legal[0] = [A - 1]                       # one legal action that is not a prefix
        legal[-1] = sorted({A - 1, A // 2})
    noises = [rng.dirichlet([0.3] * len(l)).astype(np.float32).tolist() for l in legal] if noise else None
    if players == "1p":
        tp = [-1] * B
    elif players == "2p":
        tp = rng.integers(1, 3, B).tolist()
    else:
        tp = rng.choice([-1, 1, 2], B).tolist()
        tp[0], tp[-1] = -1, 1
    return o.latent_state, o.policy_logits.cpu().numpy(), legal, noises, [int(x) for x in tp]


def _prepare(roots, logits, noises, tp):
    B = len(tp)
    if noises is None:
        roots.prepare_no_noise([0.] * B, logits, tp)
    else:
        roots.prepare(0.25, noises, [0.] * B, logits, tp)


def debug_rng(tree):
    from lightzero_b200 import cabi
    key = np.zeros(2, np.uint64)
    step = np.zeros(1, np.uint32)
    cabi.check(tree.lib.lz_tree_debug_rng(tree.h, key.ctypes.data, key[1:].ctypes.data, step.ctypes.data), "lz_tree_debug_rng")
    return int(key[0]), int(key[1])


def fused_search(cu, S, det, chance_seed, latent, logits, legal, noises, tp, cap=None, roots=None, discount=0.997,
                 delta=0.01):
    import lightzero_b200 as lzb
    mcts = lzb.StochasticMuZeroMCTSCtree(dict(num_simulations=S, deterministic=det, chance_seed=chance_seed,
                                              discount_factor=discount, value_delta_max=delta))
    if roots is None:
        roots = mcts.roots(len(tp), legal, cu.chance_space_size)
    _prepare(roots, logits, noises, tp)
    if cap is not None:
        roots._materialize(cap)
    mcts.search(roots, cu, latent, tp)
    return readout(roots, cu.action_space_size, S), debug_rng(roots._tree), roots


def oracle_search(cu, S, det, chance_seed, latent, logits, legal, noises, tp, key, variant=0, chance_variant=0,
                  discount=0.997, delta=0.01):
    """The reference loop (mcts_ctree_stochastic.py:117-252) on the C oracle with the CUDA network evaluating the leaves;
    decision ties and unpinned chance draws in hash mode with key = (seed, epoch) from step 0"""
    from oracle import ctree_port_stoch as port
    c = dict(B=len(tp), A=cu.action_space_size, C=cu.chance_space_size, S=S, legal=legal, root_logits=logits,
             noises=noises, to_play=tp, discount=discount, delta=delta, chance_seed=chance_seed)

    def setup(r):
        r.set_tie_hash(key[0], key[1], 0, variant)
        r.set_chance_variant(chance_variant)
    trace, roots = drive(port, c, "stoch", network(cu, latent, stochastic=True), det=det, setup=setup)
    return trace, roots.tie_stats()


def idle_ctas(is_chance):
    """(simulation, CTA) pairs with no selected row, for the `after` program (it runs the chance leaves) and the `rec`
    program (the others)"""
    after = rec = 0
    for lo in range(0, is_chance.shape[1], CTA_ROWS):
        blk = is_chance[:, lo:lo + CTA_ROWS].astype(bool)
        after += int((~blk.any(1)).sum())
        rec += int(blk.all(1).sum())
    return after, rec


def differ(a, b):
    """per root: different visit counts, root value or trajectory"""
    return ((a["distributions"] != b["distributions"]).any(1) | (a["root_values_bits"] != b["root_values_bits"])
            | (a["trajectories"] != b["trajectories"]).any(1))


def _report(name, st, idle, seconds):
    print(f"\n[stochastic-oracle] {name}: chance_draws={st['chance']} tie_draws={st['draws']} ties={st['ties']} "
          f"near={st['near']} max_len={st['max_len']} idle_ctas(after,rec)={idle} {seconds:.1f}s")


# ------------------------------------------------------------------------------------------------ the case matrix
PINNED = 4242
# name: config, B, S, deterministic, chance_seed, players, model mutation, input kwargs, tree capacity
CASES = {
    "cartpole_b7_det_pinned": ("cartpole", 7, 30, True, PINNED, "1p", None, {}, None),
    "cartpole_b65_det_sampled": ("cartpole", 65, 30, True, None, "1p", None, {}, None),
    "cartpole_b131_sto_pinned_2p": ("cartpole", 131, 30, False, PINNED, "2p", None, {}, None),
    "cartpole_b1201_sto_sampled": ("cartpole", 1201, 20, False, None, "1p", None, {}, None),
    "lunarlander_b65_sto_sampled_mixed": ("lunarlander_disc", 65, 40, False, None, "mixed", None, {}, None),
    "lunarlander_b131_det_pinned_2p": ("lunarlander_disc", 131, 30, True, PINNED, "2p", None, dict(noise=False), None),
    "pendulum_b65_sto_sampled_zero_policy": ("pendulum_cont_disc", 65, 40, False, None, "1p", zero_policy, dict(noise=False),
                                             None),
    "l64_c9_b131_sto_sampled_near_ties": ("l64_c9_res", 131, 30, False, None, "2p", near_policy, dict(noise=False), None),
    "l256_c608_b65_sto_sampled": ("l256_c608", 65, 20, False, None, "1p", None, {}, None),
    "l256_c608_b7_det_pinned_zero_policy": ("l256_c608", 7, 30, True, PINNED, "mixed", zero_policy, dict(noise=False), None),
    "l32_c1_b65_sto_sampled": ("l32_c1_h1", 65, 30, False, None, "1p", None, {}, None),
    "a40_c5_b131_sto_sampled_zero_policy": ("a40_c5", 131, 30, False, None, "1p", zero_policy, dict(noise=False), None),
    "a40_c5_b65_det_pinned": ("a40_c5", 65, 30, True, PINNED, "2p", None, {}, None),
    "a40_c5_b1_sto_sampled": ("a40_c5", 1, 30, False, None, "1p", None, {}, None),
    "a1_c1_b3_s200_sto_sampled": ("a1_c1", 3, 200, False, None, "1p", None, dict(masks=False), None),
    "cartpole_b64x132p37_s4_sto_sampled": ("cartpole", 64 * 132 + 37, 4, False, None, "1p", None, {}, None),
    "cartpole_b65_sto_sampled_cap300": ("cartpole", 65, 30, False, None, "2p", None, {}, 300),
}


@pytest.mark.parametrize("name", list(CASES))
def test_fused_search_equals_oracle_driving_the_same_network(name):
    cfg, B, S, det, chance_seed, players, mutate, ikw, cap = CASES[name]
    t0 = time.time()
    cu = make(cfg, mutate)
    A, C = cu.action_space_size, cu.chance_space_size
    latent, logits, legal, noises, tp = _inputs(cu, B, sum(map(ord, name)), players, **ikw)
    got, key, roots = fused_search(cu, S, det, chance_seed, latent, logits, legal, noises, tp, cap=cap)
    exp, st = oracle_search(cu, S, det, chance_seed, latent, logits, legal, noises, tp, key)
    roots.clear()
    idle = idle_ctas(exp["is_chance"])
    _report(name, st, idle, time.time() - t0)
    assert_same(got, exp)
    assert bool((np.maximum(got["distributions"], 0).sum(1) == S).all())
    # the branches the case is named for
    if C > 1:
        assert st["chance"] > 0
    if not det and A > 1:
        assert st["draws"] > 0
    if B == CTA_ROWS + 1:
        assert min(idle) > 0            # the one-row second CTA is idle in one program or the other at every simulation
    elif B > CTA_ROWS:
        assert max(idle) > 0
    if "near" in name:
        assert st["near"] > 0
    if "zero_policy" in name and A > 1:
        assert st["ties"] >= B * S // 8
    if name.startswith("a1_c1"):
        assert st["max_len"] == S           # the back-up crosses more than six 32-entry path chunks
    if C > 1 and chance_seed is None:
        assert len(np.unique(exp["last_action"][exp["is_chance"] == 0])) > 1         # the draws pick several outcomes


def test_discount_and_value_delta_max():
    """discount 0.9 with value_delta_max 0.05 in the sampled default mode; the default parameters give other searches"""
    cu = make("lunarlander_disc")
    S = 30
    latent, logits, legal, noises, tp = _inputs(cu, 131, 61, "2p")
    got, key, roots = fused_search(cu, S, False, None, latent, logits, legal, noises, tp, discount=0.9, delta=0.05)
    roots.clear()
    exp, st = oracle_search(cu, S, False, None, latent, logits, legal, noises, tp, key, discount=0.9, delta=0.05)
    default, _ = oracle_search(cu, S, False, None, latent, logits, legal, noises, tp, key)
    _report("lunarlander_b131_discount0.9_delta0.05", st, idle_ctas(exp["is_chance"]), 0.0)
    assert_same(got, exp)
    assert differ(got, default).any()
    assert st["chance"] > 0 and st["draws"] > 0


def test_large_scalars_and_value_delta_max():
    """value and reward scalars above 10^3 with value_delta_max 0.5"""
    cu = make("cartpole", large_scalars)
    S = 30
    latent, logits, legal, noises, tp = _inputs(cu, 65, 62, "1p")
    got, key, roots = fused_search(cu, S, False, None, latent, logits, legal, noises, tp, delta=0.5)
    roots.clear()
    exp, st = oracle_search(cu, S, False, None, latent, logits, legal, noises, tp, key, delta=0.5)
    o = cu.recurrent_inference(latent, torch.zeros(65, dtype=torch.int32, device="cuda"), False, return_scalars=True)
    _report("cartpole_b65_large_scalars_delta0.5", st, idle_ctas(exp["is_chance"]), 0.0)
    assert float(o.value_scalar.abs().min()) > 1e3 and float(o.reward_scalar.abs().min()) > 1e3
    assert_same(got, exp)
    assert st["chance"] > 0


def test_repeated_sampled_searches_on_one_pooled_tree():
    """Two sampled searches on one pooled tree with capacity above S: the second runs at the next epoch, equals the oracle
    there and differs from the first"""
    import lightzero_b200 as lzb
    cu = make("l64_c9_res", zero_policy)
    S, B = 25, 131
    latent, logits, legal, noises, tp = _inputs(cu, B, 63, "1p", noise=False)
    roots = lzb.StochasticMuZeroMCTSCtree.roots(B, legal, cu.chance_space_size)
    first, key1, roots = fused_search(cu, S, False, None, latent, logits, legal, noises, tp, cap=2 * S, roots=roots)
    handle = roots._tree
    second, key2, roots = fused_search(cu, S, False, None, latent, logits, legal, noises, tp, cap=2 * S, roots=roots)
    assert roots._tree is handle and handle.max_sims >= 2 * S and key2[0] == key1[0] and key2[1] > key1[1]
    roots.clear()
    for got, key in ((first, key1), (second, key2)):
        exp, st = oracle_search(cu, S, False, None, latent, logits, legal, noises, tp, key)
        assert_same(got, exp)
    _report("l64_c9_b131_repeated_cap50", st, idle_ctas(exp["is_chance"]), 0.0)
    assert differ(first, second).mean() > 0.5


def test_collect_step_equals_oracle():
    """StochasticMuZeroCollectPolicy.search_batch (sampled chance draws, hashed ties, C > A, masked roots, noise) against
    the oracle at the epoch the collect's reset produced"""
    import lightzero_b200 as lzb
    from lightzero_b200 import mz_tree
    cu = make("cartpole")
    A, C, B, S = cu.action_space_size, cu.chance_space_size, 97, 25
    rng = np.random.default_rng(64)
    obs = torch.from_numpy(rng.uniform(-1, 1, (B, cu.observation_shape)).astype(np.float32)).cuda()
    mask = (rng.random((B, A)) < 0.6).astype(np.uint8)
    mask[np.arange(B), rng.integers(0, A, B)] = 1
    mask[0] = [0, 1]
    noises = np.zeros((B, A), np.float32)
    for b in range(B):
        noises[b, :int(mask[b].sum())] = rng.dirichlet([0.3] * int(mask[b].sum()))
    pol = lzb.StochasticMuZeroCollectPolicy(cu, dict(num_simulations=S, deterministic=False, chance_seed=None,
                                                     discount_factor=0.997))
    got = pol.search_batch(obs, torch.from_numpy(mask).cuda(), torch.from_numpy(noises).cuda(), None, read_back=False)
    t = mz_tree.acquire_tree(torch.device("cuda", torch.cuda.current_device()), B, max(A, C), S)
    try:
        key = debug_rng(t)
    finally:
        t.release()
    o = cu.initial_inference(obs)
    legal = [np.nonzero(m)[0].tolist() for m in mask]
    nz = [noises[b, :len(l)].tolist() for b, l in enumerate(legal)]
    exp, st = oracle_search(cu, S, False, None, o.latent_state, o.policy_logits.cpu().numpy(), legal, nz, [-1] * B, key)
    _report("collect_cartpole_b97_sampled_masked", st, idle_ctas(exp["is_chance"]), 0.0)
    visits = got["visits"].cpu().numpy()
    assert np.array_equal(visits[:, :A], exp["distributions"]) and (visits[:, A:] == -1).all()
    assert np.array_equal(got["values"].cpu().numpy().view(np.uint32), exp["root_values_bits"])
    assert st["chance"] > 0 and st["draws"] > 0


def test_sensitivity_of_the_stochastic_comparison():
    """Oracle mutants the comparison must catch on tie- and chance-rich roots (the device is unchanged): the chance key at
    epoch + 1, step + 1 and depth - 1, the modulo draw h % C in place of the inverse CDF, the first tie always and the tie after
    the drawn one.  Each must disagree with the device on nearly every root; the default mode must also disagree with the
    pinned mode."""
    cu = make("a40_c5", zero_policy)
    S, B = 100, 132         # about 24 legal root actions: most descents past the first 24 meet tied decision nodes at depth 2
    latent, logits, legal, noises, tp = _inputs(cu, B, 65, "1p", noise=False)
    got, key, roots = fused_search(cu, S, False, None, latent, logits, legal, noises, tp)
    roots.clear()
    exp, st = oracle_search(cu, S, False, None, latent, logits, legal, noises, tp, key)
    assert_same(got, exp)
    assert st["chance"] > B and st["draws"] > B

    def frac(**kw):
        return float(differ(got, oracle_search(cu, S, False, None, latent, logits, legal, noises, tp, key, **kw)[0]).mean())
    fr = {"chance epoch+1": frac(chance_variant=1), "chance step+1": frac(chance_variant=2),
          "chance depth-1": frac(chance_variant=3), "chance h%C": frac(chance_variant=4),
          "ties[0]": frac(variant=1), "ties[(r+1)%n]": frac(variant=2)}
    pinned, _, roots = fused_search(cu, S, False, PINNED, latent, logits, legal, noises, tp)
    roots.clear()
    fr["pinned vs sampled"] = float(differ(got, pinned).mean())
    print("\n[stochastic-oracle] sensitivity, fraction of roots that disagree: " +
          ", ".join(f"{k} {v:.3f}" for k, v in fr.items()))
    assert min(fr.values()) > 0.9, fr
