"""The ReZero reanalyze sweep (``compute_target_policy_reanalyzed_rezero``, ``lz_rezero_reanalyze``) against the
reference's own loop, bit for bit.

The oracle restates ``ReZeroMZGameBuffer._compute_target_policy_reanalyzed`` (lzero/mcts/buffer/game_buffer_rezero_mz.py:194-404;
ReZeroEZGameBuffer, game_buffer_rezero_ez.py:126-330): initial_inference in mini_infer_size slices, ``compute_all_filters`` into
position groups (last position first), a plain search, then search_with_reuse walking backward with the previous search's
``get_values()`` as reuse values, and the Python target assembly.  Every search runs on the compiled reference trees through
oracle/tree_drive.py (the MuZero tree linked with the rand() == 0 shim, whose reuse descents take the first maximum; the shimmed
EfficientZero tree), with the same CUDA network evaluating the leaves it picks.  The device sweep must give identical targets,
stored child visits, root-value bits and per-simulation inference counts.
"""
import zlib

import numpy as np
import pytest
import torch

import board_model_ref as BR
import mlp_ez_model_ref as ER
import mlp_fp32_model_ref as FR
import mlp_mz_model_ref as MR
from oracle.tree_drive import drive, network

pytestmark = pytest.mark.gpu

DISCOUNT = 0.997


def _ref_trees():
    from oracle import build_ref
    mz = build_ref.load_rand0()
    import importlib.machinery
    import importlib.util
    path = build_ref.ref_module_path("ez_tree")
    ez = None
    try:
        loader = importlib.machinery.ExtensionFileLoader("ez_tree", path)
        spec = importlib.util.spec_from_file_location("ez_tree", path, loader=loader)
        ez = importlib.util.module_from_spec(spec)
        loader.exec_module(ez)
    except (ImportError, FileNotFoundError):
        ez = None
    return mz, ez


@pytest.fixture(scope="module")
def ref_trees():
    mz, ez = _ref_trees()
    if mz is None or ez is None:
        pytest.skip("compiled reference trees (oracle/_ref) not built")
    return mz, ez


# ------------------------------------------------------------------------------------------------ models of every shipped family
def _conv_sd(obs, A, seed, ez=False):
    from oracle import model_ref as R
    ref = R.EfficientZeroModelRef(obs, A) if ez else R.MuZeroModelRef(obs, A)
    return R.emulate_trained_(ref, seed).state_dict()


def make_model(family):
    """-> (model, observation shape, A, EfficientZero?, two players?, scatter by legal action?)"""
    import lightzero_b200 as lzb
    if family in ("atari_mz6", "atari_mz18"):
        A = 6 if family == "atari_mz6" else 18
        m = lzb.MuZeroModel(observation_shape=(4, 64, 64), action_space_size=A, downsample=True)
        return m.load_state_dict(_conv_sd((4, 64, 64), A, 3)), (4, 64, 64), A, False, False, False
    if family == "atari_ez":
        m = lzb.EfficientZeroModel(observation_shape=(4, 64, 64), action_space_size=6, downsample=True)
        return m.load_state_dict(_conv_sd((4, 64, 64), 6, 4, ez=True)), (4, 64, 64), 6, True, False, False
    if family in ("connect4", "gomoku"):
        m = lzb.MuZeroModel(**BR.model_kwargs(family)).load_state_dict(BR.build(family, 5).state_dict())
        return m, tuple(BR.BOARD_CONFIGS[family][0]), BR.BOARD_CONFIGS[family][1], False, True, True
    if family == "cartpole":
        m = lzb.MuZeroModelMLP(**FR.model_kwargs("cartpole")).load_state_dict(FR.build("cartpole", 6).state_dict())
        return m, (FR.CONFIGS["cartpole"][0],), FR.CONFIGS["cartpole"][1], False, False, False
    if family == "lunarlander_mz":
        m = lzb.MuZeroModelMLP(**MR.model_kwargs("lunarlander")).load_state_dict(MR.build("lunarlander", 7).state_dict())
        return m, (MR.CONFIGS["lunarlander"][0],), MR.CONFIGS["lunarlander"][1], False, False, False
    if family == "lunarlander_ez":
        m = lzb.EfficientZeroModelMLP(**ER.model_kwargs("lunarlander")).load_state_dict(ER.build("lunarlander", 8).state_dict())
        return m, (ER.CONFIGS["lunarlander"][0],), ER.CONFIGS["lunarlander"][1], True, False, False
    raise KeyError(family)


# ------------------------------------------------------------------------------------------------ inputs
def make_inputs(N, L, obs_shape, A, seed, two_player, masks, pad):
    """Rows segment * L + position.  With pad, segments end inside the window: their later rows are padding (zero
    observation, policy_mask 0, true action -2, every action legal); the last real step of a segment has true action -2."""
    rng = np.random.default_rng(seed)
    rows = N * L
    obs = torch.from_numpy(rng.random((rows,) + tuple(obs_shape), dtype=np.float32))
    mask = np.ones((rows, A), np.uint8)
    if masks:
        for i in range(rows):
            m = rng.random(A) < 0.5
            if not m.any():
                m[rng.integers(A)] = True
            mask[i] = m
        mask[0] = 0                       # a root with a single legal action (not a prefix)
        mask[0, A - 1] = 1
    tp = rng.integers(1, 3, rows).astype(np.int32) if two_player else np.full(rows, -1, np.int32)
    ta = np.asarray([rng.choice(np.nonzero(mask[i])[0]) for i in range(rows)], np.int32)
    pm = np.ones(rows, np.uint8)
    for n in range(N):
        end = int(rng.integers(1, L)) if pad and n % 2 == 0 and L > 1 else L      # real steps of this segment in the window
        ta[n * L + end - 1] = -2
        for p in range(end, L):
            i = n * L + p
            pm[i], ta[i] = 0, -2
            obs[i] = 0.0
            mask[i] = 1
    noises = np.zeros((rows, A), np.float32)
    for i in range(rows):
        noises[i] = rng.dirichlet([0.3] * A).astype(np.float32)
    pos = rng.integers(0, 50, N).tolist()
    return obs, mask, tp, ta, pm, noises, pos


# ------------------------------------------------------------------------------------------------ the reference loop
@torch.no_grad()
def oracle_sweep(ref_trees, model, ez, obs, mask, tp, ta, pm, noises, pos, L, S, A, scatter, use_noise, reuse, mini, H=5):
    rows = obs.shape[0]
    N = rows // L
    lat, logit = [], []
    for beg in range(0, rows, mini):                                # game_buffer_rezero_mz.py:243-262
        o = model.initial_inference(obs[beg:beg + mini].cuda())
        lat.append(o.latent_state)
        logit.append(o.policy_logits)
    lat, logit = torch.cat(lat), torch.cat(logit).cpu().numpy()
    mod = ref_trees[1] if ez else ref_trees[0]
    temp_values, temp_distributions, counts = [], [], []
    iter_values = None
    for it in range(L):                                             # compute_all_filters: position L - 1 - it of every segment
        idx = [i for i in range(rows) if (i + 1) % L == (L - it) % L]
        legal = [np.nonzero(mask[i])[0].tolist() for i in idx]
        c = dict(B=N, A=A, S=S, legal=legal, root_logits=logit[idx], to_play=tp[idx], use_noise=int(use_noise),
                 noises=noises[idx], discount=DISCOUNT, lstm_horizon_len=H)
        kind = "ez" if ez else "mz"
        if reuse and it > 0:
            c.update(true_action=ta[idx], reuse_value=np.asarray(iter_values, np.float32))
            kind = "ez_reuse" if ez else "reuse"
        hidden = None
        if ez:
            Hh = model.lstm_hidden_size
            hidden = (torch.zeros(N, Hh, device="cuda"), torch.zeros(N, Hh, device="cuda"))
        trace, _ = drive(mod, c, kind, network(model, lat[idx], hidden), det=True)
        if kind in ("reuse", "ez_reuse"):
            counts.append(trace["n_inferred"])
        iter_values = trace["root_values_bits"].view(np.float32).tolist()
        dist = [[int(v) for v in row if v >= 0] for row in trace["distributions"]]
        temp_values.append(iter_values)
        temp_distributions.append(dist)
    temp_values.reverse()
    temp_distributions.reverse()
    roots_values, roots_distributions = [], []
    [roots_values.extend(column) for column in zip(*temp_values)]
    [roots_distributions.extend(column) for column in zip(*temp_distributions)]
    child_visits, root_values = [dict() for _ in pos], [dict() for _ in pos]
    targets = []
    policy_index = 0
    for state_index, child_visit, root_value in zip(pos, child_visits, root_values):
        target_policies = []
        for current_index in range(state_index, state_index + L):
            distributions = roots_distributions[policy_index]
            if pm[policy_index] == 0:
                target_policies.append([0 for _ in range(A)])
            else:
                sim_num = sum(distributions)
                child_visit[current_index] = [v / sim_num for v in distributions]
                root_value[current_index] = roots_values[policy_index]
                policy = [v / sim_num for v in distributions]
                if scatter:
                    tmp = [0 for _ in range(A)]
                    for index, legal_action in enumerate(np.nonzero(mask[policy_index])[0].tolist()):
                        tmp[legal_action] = policy[index]
                    policy = tmp
                target_policies.append(policy + [0.0] * (A - len(policy)))     # fixed_action_space with a mask: zero padded
            policy_index += 1
        targets.append(target_policies)
    return np.array(targets, np.float64), child_visits, root_values, np.asarray(counts, np.int32).reshape(-1, S)


def device_sweep(model, ez, obs, mask, tp, ta, pm, noises, pos, L, S, scatter, use_noise, reuse, mini, H=5):
    import lightzero_b200 as lzb
    from lightzero_b200.reanalyze import compute_target_policy_reanalyzed_rezero
    cfg = dict(num_simulations=S, deterministic=True, discount_factor=DISCOUNT)
    mcts = lzb.EfficientZeroMCTSCtree(dict(cfg, lstm_horizon_len=H)) if ez else lzb.MuZeroMCTSCtree(cfg)
    child_visits, root_values = [dict() for _ in pos], [dict() for _ in pos]
    out, stats = compute_target_policy_reanalyzed_rezero(
        model, mcts, obs, mask, tp, ta, pm, pos, L, child_visits, root_values,
        action_type="varied_action_space" if scatter else "fixed_action_space", reanalyze_noise=use_noise,
        reuse_search=reuse, mini_infer_size=mini, noises=noises)
    return out, child_visits, root_values, mcts.last_infer_count, stats


def assert_same_sweep(got, exp, S):
    out, cv, rv, cnt, stats = got
    e_out, e_cv, e_rv, e_cnt = exp
    assert out.dtype == np.float64 and out.shape == e_out.shape
    assert np.array_equal(out.view(np.uint64), e_out.view(np.uint64)), "targets differ"
    assert cv == e_cv, "stored child visits differ"
    for a, b in zip(rv, e_rv):
        assert a.keys() == b.keys()
        assert all(np.float32(a[k]).view(np.uint32) == np.float32(b[k]).view(np.uint32) for k in a), "root values differ"
    assert np.array_equal(cnt, e_cnt), "inference counts differ"
    from lightzero_b200.reanalyze import rezero_reuse_stats
    assert stats == rezero_reuse_stats(e_cnt, S)


CASES = [
    # family, N, L, S, masks, pad, noise, reuse, mini
    ("atari_mz6", 1, 1, 10, False, False, True, True, 10240),
    ("atari_mz6", 7, 2, 10, False, True, True, True, 10240),
    ("atari_mz6", 7, 6, 12, False, True, True, True, 16),
    ("atari_mz6", 256, 6, 10, False, True, True, True, 512),
    ("atari_mz6", 256, 2, 10, False, True, False, True, 10240),
    ("atari_mz6", 7, 6, 10, False, True, True, False, 10240),
    ("atari_mz6", 1024, 5, 8, False, True, True, True, 2048),
    ("atari_mz18", 7, 6, 12, True, True, True, True, 10240),
    ("atari_ez", 7, 6, 10, False, True, True, True, 10240),
    ("atari_ez", 256, 2, 8, False, True, False, True, 100),
    ("atari_ez", 1, 6, 8, False, False, True, False, 10240),
    ("connect4", 7, 6, 12, True, True, True, True, 10240),
    ("gomoku", 256, 2, 10, True, True, True, True, 10240),
    ("gomoku", 1, 6, 10, True, False, False, True, 10240),
    ("cartpole", 7, 6, 12, False, True, True, True, 10240),
    ("cartpole", 256, 1, 10, False, True, True, True, 10240),
    ("lunarlander_mz", 7, 6, 12, False, True, True, True, 10240),
    ("lunarlander_mz", 256, 2, 10, False, True, False, True, 10240),
    ("lunarlander_ez", 7, 6, 12, False, True, True, True, 10240),
    ("lunarlander_ez", 1, 2, 10, False, True, True, False, 10240),
]


@pytest.mark.parametrize("family, N, L, S, masks, pad, noise, reuse, mini", CASES,
                         ids=[f"{c[0]}-N{c[1]}-L{c[2]}-S{c[3]}" + "-mask" * c[4] + "-pad" * c[5] + "-nonoise" * (not c[6]) +
                              "-noreuse" * (not c[7]) + f"-mini{c[8]}" for c in CASES])
def test_sweep_matches_reference_loop(ref_trees, family, N, L, S, masks, pad, noise, reuse, mini):
    model, obs_shape, A, ez, two_player, scatter = make_model(family)
    args = make_inputs(N, L, obs_shape, A, zlib.crc32(f"{family}-{N}-{L}".encode()) % 1000, two_player, masks, pad)
    got = device_sweep(model, ez, *args, L, S, scatter, noise, reuse, mini)
    exp = oracle_sweep(ref_trees, model, ez, *args, L, S, A, scatter, noise, reuse, mini)
    assert_same_sweep(got, exp, S)
    if pad:
        assert (args[4] == 0).any() or L == 1
    print(f"{family} N={N} L={L}: stats {got[4]}")


def test_fixed_action_space_with_masks_pads_zeros(ref_trees):
    """fixed_action_space on masked roots: the legal-order distribution, zero padded"""
    model, obs_shape, A, ez, _, _ = make_model("atari_mz6")
    args = make_inputs(7, 3, obs_shape, A, 21, False, True, True)
    got = device_sweep(model, ez, *args, 3, 10, False, True, True, 10240)
    exp = oracle_sweep(ref_trees, model, ez, *args, 3, 10, A, False, True, True, 10240)
    assert_same_sweep(got, exp, 10)


def test_second_sweep_captures_no_graph():
    from lightzero_b200 import cabi
    lib = cabi.load()
    model, obs_shape, A, ez, _, _ = make_model("atari_mz6")
    args = make_inputs(16, 4, obs_shape, A, 31, False, False, True)
    first = device_sweep(model, ez, *args, 4, 10, False, True, True, 10240)
    n0 = lib.lz_debug_graph_captures()
    second = device_sweep(model, ez, *args, 4, 10, False, True, True, 10240)
    assert lib.lz_debug_graph_captures() == n0, "the second sweep of the same shape captured a graph"
    assert np.array_equal(first[0], second[0]) and first[1] == second[1]


def test_sweep_on_side_stream_next_to_busy_default_stream():
    model, obs_shape, A, ez, _, _ = make_model("atari_mz6")
    args = make_inputs(64, 5, obs_shape, A, 41, False, False, True)
    ref = device_sweep(model, ez, *args, 5, 10, False, True, True, 10240)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    torch.cuda._sleep(200_000_000)                  # the legacy default stream stays busy while the sweep runs
    with torch.cuda.stream(side):
        got = device_sweep(model, ez, *args, 5, 10, False, True, True, 10240)
    torch.cuda.synchronize()
    assert np.array_equal(got[0].view(np.uint64), ref[0].view(np.uint64)) and got[1] == ref[1] and got[2] == ref[2]
    assert np.array_equal(got[3], ref[3])


def test_latent_inputs_equal_observation_inputs():
    """lz_rezero_reanalyze on the latents and logits of a prior initial_inference gives what it gives on the observations"""
    import lightzero_b200 as lzb
    from lightzero_b200 import cabi, mz_tree
    model, obs_shape, A, ez, _, _ = make_model("cartpole")
    N, L, S = 9, 3, 10
    obs, mask, tp, ta, pm, noises, pos = make_inputs(N, L, obs_shape, A, 51, False, False, True)
    mcts = lzb.MuZeroMCTSCtree(dict(num_simulations=S, deterministic=True))
    t = mz_tree.acquire_tree(model.device, N, A, S)
    t.set_params(*mcts._params())
    q = t.search_for(model, S)
    dev = model.device
    obs_d = obs.to(dev)
    o = model.initial_inference(obs_d)
    d = {k: torch.from_numpy(v).to(dev) for k, v in dict(mask=mask, tp=tp, ta=ta, pm=pm, nz=noises).items()}
    outs = []
    for use_obs in (True, False):
        tg = torch.empty((N, L, A), dtype=torch.float64, device=dev)
        cv = torch.empty_like(tg)
        rv = torch.empty((N, L), dtype=torch.float32, device=dev)
        ic = torch.empty((L - 1, S), dtype=torch.int32, device=dev)
        lat = o.latent_state.contiguous()
        lg = o.policy_logits.contiguous()
        cabi.check(t.lib.lz_rezero_reanalyze(
            q, L, 1, 10240, obs_d.data_ptr() if use_obs else None, None if use_obs else lat.data_ptr(),
            None if use_obs else lg.data_ptr(), d["mask"].data_ptr(), d["tp"].data_ptr(), d["ta"].data_ptr(), d["pm"].data_ptr(),
            d["nz"].data_ptr(), 0.25, 1, 0, tg.data_ptr(), rv.data_ptr(), cv.data_ptr(), ic.data_ptr(), cabi.stream_ptr()),
            "lz_rezero_reanalyze")
        outs.append([x.cpu().numpy() for x in (tg, cv, rv, ic)])
    t.release()
    for a, b in zip(*outs):
        assert np.array_equal(a, b)


def test_wrong_model_tree_pairs_raise():
    import lightzero_b200 as lzb
    from lightzero_b200.reanalyze import compute_target_policy_reanalyzed_rezero
    mz, _, A, _, _, _ = make_model("cartpole")
    ezm, _, _, _, _, _ = make_model("lunarlander_ez")
    args = (np.zeros((2, 4), np.float32), np.ones((2, A), np.uint8), [-1] * 2, [0, -2], [1, 1], [0], 2)
    with pytest.raises(TypeError):
        compute_target_policy_reanalyzed_rezero(mz, lzb.EfficientZeroMCTSCtree(dict(num_simulations=4)), *args)
    with pytest.raises(TypeError):
        compute_target_policy_reanalyzed_rezero(ezm, lzb.MuZeroMCTSCtree(dict(num_simulations=4)), *args)
    with pytest.raises(TypeError):
        compute_target_policy_reanalyzed_rezero(mz, lzb.GumbelMuZeroMCTSCtree(dict(num_simulations=4)), *args)
