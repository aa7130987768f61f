"""The fused search graph of every tree mode (csrc/search.cu, enqueue_search) and the step-wise drive of the same trees
(MuZeroMCTSCtree._search_stepwise):
- the exact kernel-node count of each mode's graph: the persistent MuZero launch, the multi-kernel MuZero graph, EfficientZero
  plain and reuse, Gumbel on the conv, board and MLP models, Stochastic MuZero on the MLP and board models;
- a Stochastic MuZero search driven step by step around a model that is not a lightzero_b200 model equals the fused search,
  bit for bit: visit counts, root-value bits and trajectories (the MLP model's root values excepted: its kernel's read-out
  differs from the step-wise drive's in the last bits)."""
import pytest

import stoch_board_model_ref as SB
import stoch_mlp_model_ref as SR
import test_gpu_board as TB
import test_gpu_ez as TE
import test_gpu_gumbel as TG
import test_gpu_search as TS
import test_gpu_stochastic as TST
import test_gpu_stochastic_board as TSB

pytestmark = pytest.mark.gpu

S = 12


def _muzero(A):
    _, cu, obs, _, legal, noises, mcts = TS._setup(16, A, S)
    out = cu.initial_inference(obs.cuda())
    roots = mcts.roots(16, legal)
    roots.prepare(0.25, noises, [0.] * 16, out.policy_logits, [-1] * 16)
    mcts.search(roots, cu, out.latent_state, [-1] * 16)
    roots.clear()
    return mcts.last_num_kernels


def _ez(reuse):
    B, A = 16, 6
    _, cu, obs, _, legal, noises, mcts = TE._setup(B, A, S, masks=True, horizon=3)
    out = cu.initial_inference(obs.cuda())
    roots = mcts.roots(B, legal)
    roots.prepare(0.25, noises, [0.] * B, out.policy_logits, [-1] * B)
    if reuse:
        true_action = [l[0] for l in legal]
        mcts.search_with_reuse(roots, cu, out.latent_state, out.reward_hidden_state, [-1] * B, true_action, [0.5] * B)
    else:
        mcts.search(roots, cu, out.latent_state, out.reward_hidden_state, [-1] * B)
    roots.clear()
    return mcts.last_num_kernels


def _gumbel(family):
    B, A = 16, 6
    if family == "conv":
        cu, obs = TG._conv_model(A, (4, 64, 64), 1), (4, 64, 64)
    elif family == "board":
        _, cu = TB.make("tictactoe", 1)
        A, obs = cu.action_space_size, tuple(TB.BR.BOARD_CONFIGS["tictactoe"][0])
    else:
        cu, obs = TG._mlp_model(A, 1), 4
    out, legal, noises = TG._roots_inputs(cu, B, A, obs, 3, True)
    _, mcts, roots = TG._fused_search(cu, out, legal, noises, B, A, S, 4)
    roots.clear()
    return mcts.last_num_kernels


def _stochastic_inputs(family, name, B, seed):
    """(model, initial inference, legal, noises, to_play, chance_space_size, support range) of a Stochastic MuZero config"""
    if family == "mlp":
        cu, o, legal, noises, to_play, C = TST.case(name, B, False, True, True, seed)
        return cu, o, legal, noises, to_play, C, SR.CONFIGS[name][6]
    cu, o, legal, noises, to_play = TSB.case(name, B, False, True, seed)
    return cu, o, legal, noises, to_play, cu.chance_space_size, SB.CONFIGS[name][7]


def _stochastic_search(model, o, legal, noises, to_play, C, sup, chance_seed):
    import lightzero_b200 as lzb
    B = len(legal)
    mcts = lzb.StochasticMuZeroMCTSCtree(dict(num_simulations=S, deterministic=True, chance_seed=chance_seed,
                                              model=dict(value_support_range=sup, reward_support_range=sup)))
    roots = mcts.roots(B, legal, C)
    roots.prepare(0.25, noises, [0.] * B, o.policy_logits, to_play)
    mcts.search(roots, model, o.latent_state, to_play)
    got = TST.readout(roots)
    roots.clear()
    return got, mcts


def _stochastic(family):
    cu, o, legal, noises, to_play, C, sup = _stochastic_inputs(family, "cartpole" if family == "mlp" else "game_2048", 16, 1)
    return _stochastic_search(cu, o, legal, noises, to_play, C, sup, 7)[1].last_num_kernels


# a persistent search is one launch; a multi-kernel graph is [descent] + S x [the model's launches, back-up (+ next descent)],
# where the EfficientZero model is 3 launches (conv trunk, LSTM GEMM, value-prefix head), the Stochastic MuZero model 2 (the
# afterstate and the dynamics program), every other model 1, and the EfficientZero reuse search adds S - 1 separate descents
GRAPHS = {
    "muzero_persistent": (lambda: _muzero(6), 1),
    "muzero_multi_kernel": (lambda: _muzero(33), 1 + 2 * S),
    "efficientzero": (lambda: _ez(False), 1 + 4 * S),
    "efficientzero_reuse": (lambda: _ez(True), 1 + 4 * S + (S - 1)),
    "gumbel_conv": (lambda: _gumbel("conv"), 1 + 2 * S),
    "gumbel_board": (lambda: _gumbel("board"), 1 + 2 * S),
    "gumbel_mlp": (lambda: _gumbel("mlp"), 1 + 2 * S),
    "stochastic_mlp": (lambda: _stochastic("mlp"), 1 + 3 * S),
    "stochastic_board": (lambda: _stochastic("board"), 1 + 3 * S),
}


@pytest.mark.parametrize("mode", list(GRAPHS))
def test_graph_kernel_count(mode):
    run, want = GRAPHS[mode]
    assert run() == want


class _Unfused:
    """Not a lightzero_b200 model: StochasticMuZeroMCTSCtree drives the device trees one simulation at a time around it."""

    def __init__(self, model):
        self.model = model

    def recurrent_inference(self, state, option, afterstate=False):
        return self.model.recurrent_inference(state, option, afterstate=afterstate)


def _stochastic_pair(family, name, B, seed):
    """(fused, step-wise) read-outs of one Stochastic MuZero search on the same inputs, chance draws pinned"""
    cu, o, legal, noises, to_play, C, sup = _stochastic_inputs(family, name, B, seed)
    fused, _ = _stochastic_search(cu, o, legal, noises, to_play, C, sup, 3000 + seed)
    step, _ = _stochastic_search(_Unfused(cu), o, legal, noises, to_play, C, sup, 3000 + seed)
    assert all(sum(d) == S for d in fused["dist"])
    return fused, step


# StochasticMuZeroModelMLP runs on mlp_tc.cu, whose read-out folds the support in quads (tests/test_gpu_scalar_readout.py):
# its values and rewards differ from lz_inverse_scalar_transform of the same logits in the last bits, and so do the root
# values of the two searches.  Strict: the mark must go when the two read-outs agree.
MLP_CASES = [("lunarlander_disc", 40, 1), ("l64_c9_res", 20, 3)]
MLP_READOUT = pytest.mark.xfail(strict=True, raises=AssertionError,
                                reason="mlp_tc.cu's quad-order read-out differs from lz_inverse_scalar_transform in the last bits")


@pytest.mark.parametrize("family,name,B,seed", [("board", "game_2048", 64, 0), ("board", "c32_6x7_a12", 40, 3)] +
                         [pytest.param("mlp", *c, marks=MLP_READOUT) for c in MLP_CASES])
def test_stochastic_stepwise_equals_fused(family, name, B, seed):
    """The step-wise drive reads values and rewards through the torch InverseScalarTransform, the fused graph through the
    network kernel's read-out: the two searches agree bit for bit"""
    fused, step = _stochastic_pair(family, name, B, seed)
    TST.assert_equal(step, fused)


@pytest.mark.parametrize("name,B,seed", MLP_CASES)
def test_stochastic_mlp_stepwise_visits_equal_fused(name, B, seed):
    """The MLP searches of test_stochastic_stepwise_equals_fused: the same visit counts and trajectories"""
    fused, step = _stochastic_pair("mlp", name, B, seed)
    assert step["dist"] == fused["dist"]
    assert step["traj"] == fused["traj"]
