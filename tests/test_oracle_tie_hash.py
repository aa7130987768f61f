"""The oracle's tie-break hash mode (oracle/ctree_port.c lzo_tree_set_tie_hash).

In hash mode a non-deterministic descent draws from the reference's tie list (cnode.cpp:576-586) with the device trees'
counter-based hash, r = mix64(seed ^ mix64(epoch) ^ mix64((b << 32) | step) ^ depth) % len(ties), instead of rand().
Given the seed, epoch and step the device used, the oracle then judges the device's stochastic searches bit for bit.

`tie_rich_case` is shared with the GPU tests (test_gpu_tree.py): quantized logits, rewards and values make exact and near
ties common at every depth."""
import numpy as np
import pytest

from oracle import ctree_port as port
from oracle import ctree_port_ez as port_ez
from oracle.tree_drive import assert_same, drive, recorded

M64 = 2 ** 64 - 1


def mix64(z):
    """splitmix64 finaliser (lightzero_b200/csrc/tree.cuh mix64), in Python integers"""
    z = (z + 0x9e3779b97f4a7c15) & M64
    z = ((z ^ (z >> 30)) * 0xbf58476d1ce4e5b9) & M64
    z = ((z ^ (z >> 27)) * 0x94d049bb133111eb) & M64
    return z ^ (z >> 31)


def tie_draw(seed, epoch, b, step, depth, n):
    return mix64(seed ^ mix64(epoch) ^ mix64(((b << 32) | step) & M64) ^ depth) % n if n > 1 else 0


def tie_rich_case(B, A, S, seed, masks=True, two_p=False):
    """Random tree inputs on a coarse grid: equal logits give equal priors, equal rewards and values equal Q values."""
    rng = np.random.default_rng(seed)
    legal = []
    for _ in range(B):
        m = rng.random(A) < 0.6 if masks else np.ones(A, bool)
        if not m.any():
            m[rng.integers(A)] = True
        legal.append(np.nonzero(m)[0].tolist())

    def q(shape, lo, hi, step):
        return (rng.integers(lo, hi + 1, shape) * step).astype(np.float32)
    return dict(B=B, A=A, S=S, legal=legal, root_logits=q((B, A), -1, 1, 0.5), rewards=q((S, B), -1, 1, 0.25),
                values_in=q((S, B), -2, 2, 0.25), policies=q((S, B, A), -1, 1, 0.5), lstm_horizon_len=3,
                to_play=(rng.integers(1, 3, B) if two_p else np.full(B, -1)).astype(np.int32).tolist(),
                true_action=[int(l[rng.integers(len(l))]) for l in legal], reuse_value=q((B,), -2, 2, 0.25).tolist())


def port_drive(kind, c, **kw):
    """tree_drive.drive on the port with the recorded outputs of case `c`"""
    mod = port_ez if kind in ("ez", "ez_reuse") else port
    return drive(mod, c, kind, recorded(c, kind), **kw)


KINDS = ["mz", "ez", "reuse", "ez_reuse"]


@pytest.mark.parametrize("two_p", [False, True])
@pytest.mark.parametrize("kind", KINDS)
def test_hash_that_draws_zero_equals_deterministic_mode(kind, two_p):
    """Hash mode with r forced to 0 takes the first tie like the deterministic rule: bit-identical traces and results.
    The unforced hash mode must leave the deterministic path on these tie-rich inputs."""
    c = tie_rich_case(64, 7, 40, 11 + two_p, two_p=two_p)
    det, _ = port_drive(kind, c, det=True)
    zero, roots = port_drive(kind, c, det=False, setup=lambda r: r.set_tie_hash(0x5eed5eed, 3, 0, variant=1))
    assert_same(zero, det)
    st = roots.tie_stats()
    assert st["ties"] > 100 and st["draws"] == 0 and st["near"] == 0
    drawn, roots = port_drive(kind, c, det=False, setup=lambda r: r.set_tie_hash(0x5eed5eed, 3, 0))
    assert roots.tie_stats()["draws"] > 50
    assert not np.array_equal(drawn["distributions"], det["distributions"])


def test_hash_draw_is_the_device_formula():
    """Roots whose children all tie: the first descent of tree b at step s takes legal[b][tie_draw(...)] (depth 0), for
    legal lists that are not a prefix and for several steps, seeds and epochs."""
    B, A = 40, 9
    rng = np.random.default_rng(5)
    legal = [sorted(rng.choice(A, size=int(rng.integers(1, A + 1)), replace=False).tolist()) for _ in range(B)]
    for seed, epoch, step0 in ((0x5eed5eed, 1, 0), (12345, 7, 3), (2 ** 64 - 1, 2 ** 40 + 5, 2 ** 31)):
        roots = port.Roots(B, legal, action_space_size=A, max_sims=8)
        roots.prepare_no_noise([0.] * B, np.zeros((B, A), np.float32).tolist(), [-1] * B)
        roots.set_tie_hash(seed, epoch, step0)
        mm = port.MinMaxStatsList(B)
        mm.set_delta(0.01)
        for k in range(4):        # no back-up: every traverse scans the same all-tied root
            _, _, la, _ = port.batch_traverse(roots, 19652, 1.25, 0.997, mm, port.ResultsWrapper(B), [-1] * B, False)
            exp = [legal[b][tie_draw(seed, epoch, b, step0 + k, 0, len(legal[b]))] for b in range(B)]
            assert la == exp, (seed, epoch, k)
        st = roots.tie_stats()
        assert st["ties"] == 4 * sum(len(l) > 1 for l in legal) and st["max_len"] == 1


def test_forced_ties_draw_every_position():
    """All children of every root tie exactly (zero logits, no noise): over 600 roots every tie position is drawn, each
    about equally often; the deterministic rule only ever takes position 0."""
    B, A = 600, 6
    roots = port.Roots(B, [list(range(A))] * B, action_space_size=A, max_sims=4)
    roots.prepare_no_noise([0.] * B, np.zeros((B, A), np.float32).tolist(), [-1] * B)
    roots.set_tie_hash(0x5eed5eed, 1, 0)
    mm = port.MinMaxStatsList(B)
    mm.set_delta(0.01)
    _, _, la, _ = port.batch_traverse(roots, 19652, 1.25, 0.997, mm, port.ResultsWrapper(B), [-1] * B, False)
    counts = np.bincount(la, minlength=A)
    assert (counts >= B / A / 2).all(), counts
    st = roots.tie_stats()
    assert st["ties"] == B and st["draws"] == B - counts[0]
    _, _, la, _ = port.batch_traverse(roots, 19652, 1.25, 0.997, mm, port.ResultsWrapper(B), [-1] * B, True)
    assert set(la) == {0}


def test_near_ties_are_counted():
    """Priors that differ by ~1e-7 give tie lists with unequal scores within the 1e-6 epsilon (cnode.cpp:583): the list
    holds the first maximum and every LATER child within epsilon, so the logits decrease along the legal list."""
    B, A = 50, 5
    logits = (np.arange(A, dtype=np.float32) * -5e-7)[None].repeat(B, 0)
    roots = port.Roots(B, [list(range(A))] * B, action_space_size=A, max_sims=4)
    roots.prepare_no_noise([0.] * B, logits.tolist(), [-1] * B)
    roots.set_tie_hash(1, 1, 0)
    mm = port.MinMaxStatsList(B)
    mm.set_delta(0.01)
    for s in range(2):      # the first descent sees exact ties (no visits yet: no prior term), the second near ties
        res = port.ResultsWrapper(B)
        _, _, _, vtp = port.batch_traverse(roots, 19652, 1.25, 0.997, mm, res, [-1] * B, False)
        port.batch_backpropagate(s + 1, 0.997, [0.] * B, [0.] * B, np.zeros((B, A), np.float32).tolist(), mm, res, vtp)
    st = roots.tie_stats()
    assert st["near"] == B and st["ties"] == 2 * B
