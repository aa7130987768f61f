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


# ---- Stochastic MuZero chance draws --------------------------------------------------------------------------------------
_LIBM = None


def expf(x):
    """glibc's expf, the one the port's expand calls"""
    global _LIBM
    if _LIBM is None:
        import ctypes
        _LIBM = ctypes.CDLL("libm.so.6")
        _LIBM.expf.restype, _LIBM.expf.argtypes = ctypes.c_float, [ctypes.c_float]
    return np.float32(_LIBM.expf(float(x)))


def priors_of(logits):
    """CNode::expand's softmax in float32, sequential in key order (ctree_stochastic_muzero cnode.cpp:143-166)"""
    logits = np.asarray(logits, np.float32)
    m = np.float32(np.max(logits))
    temp = [expf(np.float32(x - m)) for x in logits]
    s = np.float32(0.0)
    for x in temp:
        s = np.float32(s + x)
    return [np.float32(x / s) for x in temp]


def chance_u(seed, epoch, b, step, depth):
    """the uniform of a hashed chance draw: the tie hash key, >> 11, times 2^-53"""
    h = mix64(seed ^ mix64(epoch) ^ mix64(((b << 32) | step) & M64) ^ depth)
    return float(h >> 11) * 2.0 ** -53


def discrete_draw(priors, u):
    """std::discrete_distribution<>(priors) at the uniform u in libstdc++: double sum, p / sum, partial sums with the last
    set to 1.0, lower_bound; fewer than two outcomes draw 0"""
    if len(priors) < 2:
        return 0
    s = 0.0
    for p in priors:
        s += float(p)
    cp, acc = [], 0.0
    for p in priors:
        acc += float(p) / s
        cp.append(acc)
    cp[-1] = 1.0
    return int(np.searchsorted(np.asarray(cp), u, side="left"))


def _chance_chains(C, B, S, seed, key, variant=0):
    """B trees whose decision nodes have one action, so every descent alternates action 0 and a chance draw; the chance
    leaves get random logits (some far below the rest: zero priors).  Returns the port's per-simulation paths and the
    logits of every chance node, keyed by its path."""
    from oracle import ctree_port_stoch as ps
    rng = np.random.default_rng(seed)
    roots = ps.Roots(B, [[0]] * B, C, max_sims=S, action_space_size=1)
    roots.prepare_no_noise([0.] * B, np.zeros((B, 1), np.float32).tolist(), [-1] * B)
    roots.set_tie_hash(*key)
    roots.set_chance_variant(variant)
    mm = ps.MinMaxStatsList(B)
    mm.set_delta(0.01)
    nodes, paths = {}, []
    for s in range(S):
        res = ps.ResultsWrapper(B)
        ch, _, _, _, vtp = ps.batch_traverse(roots, 19652, 1.25, 0.997, mm, res, [-1] * B, False)
        traj = roots.get_trajectories()
        paths.append(traj)
        logits = (rng.standard_normal((B, C)) * 2).astype(np.float32)
        logits[rng.random((B, C)) < 0.2] = -200.0
        for b in range(B):
            if ch[b]:
                nodes[(b,) + tuple(traj[b])] = logits[b]
        pol = [logits[b].tolist() if ch[b] else [0.0] for b in range(B)]
        ps.batch_backpropagate(s + 1, 0.997, rng.standard_normal(B).tolist(), rng.standard_normal(B).tolist(), pol, mm, res,
                               vtp, ch, list(range(B)))
    return paths, nodes, roots.tie_stats()


@pytest.mark.parametrize("C", [2, 7, 40])
def test_chance_draw_is_the_device_formula(C):
    """Hash mode (no pinned u): every chance outcome of the port is lower_bound(partial sums of the node's priors, u) with
    u = (mix64(seed ^ mix64(epoch) ^ mix64((b << 32) | step) ^ depth) >> 11) * 2^-53, restated here in Python, for every
    (tree, step, depth) of a few thousand draws; the chance draw counter counts them"""
    B, S, key = 150, 14, (0xdeadbeefcafe, 5, 3)
    paths, nodes, st = _chance_chains(C, B, S, 100 + C, key)
    n = 0
    for s, traj in enumerate(paths):
        for b in range(B):
            for d in range(1, len(traj[b]), 2):
                pri = priors_of(nodes[(b,) + tuple(traj[b][:d])])
                assert traj[b][d] == discrete_draw(pri, chance_u(key[0], key[1], b, key[2] + s, d)), (b, s, d)
                n += 1
    assert n > 2000 and st["chance"] == n and st["ties"] == 0
    assert max(len(t) for p in paths for t in p) >= 5


@pytest.mark.parametrize("variant", [1, 2, 3, 4])
def test_chance_draw_mutants_change_the_outcomes(variant):
    """The sensitivity mutants of the chance key (epoch + 1, step + 1, depth - 1) and the modulo draw h % C give other
    outcomes on most draws where the priors leave a choice"""
    C, B, S, key = 5, 150, 8, (77, 2, 0)
    base, _, _ = _chance_chains(C, B, S, 7, key)
    mut, _, _ = _chance_chains(C, B, S, 7, key, variant)
    first = [next((s for s in range(S) if base[s][b] != mut[s][b]), None) for b in range(B)]
    assert sum(f is not None for f in first) > 0.8 * B, variant
