"""The case grid of the replay buffer's reward / value targets (``reanalyze.compute_target_reward_value``), shared by the fixture
generator (tests/golden/make_value_targets_golden.py), the CPU tests and the GPU tests.

``make_context(case)`` builds a ``reward_value_context`` the way ``MuZeroGameBuffer._prepare_reward_value_context``
(lzero/mcts/buffer/game_buffer_muzero.py:291-360) does from sampled game segments: per segment a length, a position inside it,
a reward segment padded past the end by up to td - 1 steps (as GameSegment.pad_over does), td clipped to the steps left, and
value_mask 1 where the bootstrap index is inside the segment.  Everything is drawn from the case's seed.
"""
import zlib

import numpy as np

# name -> dict(kind 'mz' | 'ez', N, K1, td, discount, rewards 'f32' | 'f64' | 'f32x1' | 'f64x1', players 1 | 2, H, root)
CASES = {
    "mz_f32_n1_k6": dict(kind="mz", N=1, K1=6, td=5, discount=0.997, rewards="f32", players=1),
    "mz_f32_n7_k6": dict(kind="mz", N=7, K1=6, td=5, discount=0.997, rewards="f32", players=1),
    "mz_f64_n7_k6": dict(kind="mz", N=7, K1=6, td=5, discount=0.997, rewards="f64", players=1),
    "mz_f32x1_n7_k6": dict(kind="mz", N=7, K1=6, td=5, discount=0.997, rewards="f32x1", players=1),
    "mz_f32_n64_k6_td1": dict(kind="mz", N=64, K1=6, td=1, discount=0.997, rewards="f32", players=1),
    "mz_f32_n64_k6_td9": dict(kind="mz", N=64, K1=6, td=9, discount=0.997, rewards="f32", players=1),
    "mz_f64_n64_k6_td9_d1": dict(kind="mz", N=64, K1=6, td=9, discount=1.0, rewards="f64", players=1),
    "mz_f32_n64_k1": dict(kind="mz", N=64, K1=1, td=5, discount=0.997, rewards="f32", players=1),
    "mz_f32_n7_k6_d1": dict(kind="mz", N=7, K1=6, td=5, discount=1.0, rewards="f32", players=1),
    "mz_2p_f32_n64_k6": dict(kind="mz", N=64, K1=6, td=5, discount=0.997, rewards="f32", players=2),
    "mz_2p_f64_n7_k6_td9": dict(kind="mz", N=7, K1=6, td=9, discount=1.0, rewards="f64", players=2),
    "mz_2p_f32_n7_k1_td1": dict(kind="mz", N=7, K1=1, td=1, discount=0.997, rewards="f32", players=2),
    "ez_f32_n7_k6_h5": dict(kind="ez", N=7, K1=6, td=5, discount=0.997, rewards="f32", players=1, H=5),
    "ez_f64_n7_k6_h5": dict(kind="ez", N=7, K1=6, td=5, discount=0.997, rewards="f64", players=1, H=5),
    "ez_f32x1_n7_k6_h5": dict(kind="ez", N=7, K1=6, td=5, discount=0.997, rewards="f32x1", players=1, H=5),
    "ez_f64x1_n7_k6_h1": dict(kind="ez", N=7, K1=6, td=5, discount=0.997, rewards="f64x1", players=1, H=1),
    "ez_f32_n64_k6_h1_td9": dict(kind="ez", N=64, K1=6, td=9, discount=0.997, rewards="f32", players=1, H=1),
    "ez_f32_n64_k6_h5_td1_d1": dict(kind="ez", N=64, K1=6, td=1, discount=1.0, rewards="f32", players=1, H=5),
    "ez_f32_n1_k1_h5": dict(kind="ez", N=1, K1=1, td=5, discount=0.997, rewards="f32", players=1, H=5),
    "ez_f32_n64_k1_h5": dict(kind="ez", N=64, K1=1, td=5, discount=0.997, rewards="f32", players=1, H=5),
    "ez_2p_f32_n64_k6_h5": dict(kind="ez", N=64, K1=6, td=5, discount=0.997, rewards="f32", players=2, H=5),
    "ez_2p_f32x1_n7_k6_h5_td9": dict(kind="ez", N=7, K1=6, td=9, discount=1.0, rewards="f32x1", players=2, H=5),
    "ez_root_f32_n7_k6_h5": dict(kind="ez", N=7, K1=6, td=5, discount=0.997, rewards="f32", players=1, H=5, root=True),
    "ez_root_2p_f32_n7_k6_h5": dict(kind="ez", N=7, K1=6, td=5, discount=0.997, rewards="f32", players=2, H=5, root=True),
}
# MuZeroGameBuffer with use_root_value=True: the reference fails (np.array of an empty list times the td discounts)
MZ_ROOT_FAILURE = dict(kind="mz", N=7, K1=6, td=5, discount=0.997, rewards="f32", players=1, root=True)


def seed_of(name):
    return zlib.crc32(name.encode()) % 100000


def make_context(case, seed, A=6):
    """-> dict: value_mask, pos, rewards_list, game_segment_lens, td_steps_list, to_play_segment, env_type, values (fp32 [T], the
    stand-in network's value scalars), root_values (fp32 [T]), action_mask [T, A], to_play [T] (as
    _preprocess_to_play_and_action_mask builds them) and noises [T, A]."""
    rng = np.random.default_rng(seed)
    N, K1, td_cfg = case["N"], case["K1"], case["td"]
    dtype = np.float64 if case["rewards"].startswith("f64") else np.float32
    column = case["rewards"].endswith("x1")
    two = case["players"] == 2
    value_mask, td_steps_list, pos, lens, rewards_list, to_play_segment, action_mask_segment = [], [], [], [], [], [], []
    for n in range(N):
        gsl = int(rng.integers(1, 3 * K1 + 2 * td_cfg + 2))
        # segments that end inside the unroll and inside the td window, and segments ending exactly at the position
        s = int(rng.integers(max(0, gsl - K1 - td_cfg - 1), gsl)) if n % 3 else int(rng.integers(0, gsl))
        pad = int(rng.integers(0, td_cfg)) if n % 2 else 0
        r = rng.normal(0, 2, gsl + pad)
        r[rng.random(r.shape) < 0.15] = 0.0
        r[rng.random(r.shape) < 0.1] = -0.0
        m = rng.random(r.shape) < 0.2
        r[m] = rng.integers(-3, 4, int(m.sum()))
        r = r.astype(dtype)
        if column:
            r = r.reshape(-1, 1)
        rewards_list.append(r)
        # to_play runs K1 steps past the rewards: EfficientZero's base_index can move past the segment's end
        if two:
            first = int(rng.integers(1, 3))
            tp = np.array([first if i % 2 == 0 else 3 - first for i in range(gsl + pad + K1)], np.int64)
        else:
            tp = np.full(gsl + pad + K1, -1, np.int64)
        to_play_segment.append(tp)
        am = (rng.random((gsl + pad, A)) < 0.6).astype(np.int8)
        am[np.arange(gsl + pad), rng.integers(0, A, gsl + pad)] = 1
        action_mask_segment.append(am)
        td = np.clip(td_cfg, 1, max(1, gsl - s)).astype(np.int32)
        for c in range(s, s + K1):
            td_steps_list.append(td)
            value_mask.append(1 if c + td < gsl else 0)
        pos.append(s)
        lens.append(gsl)
    T = N * K1
    values = (rng.normal(0, 3, T)).astype(np.float32)
    m = rng.random(T) < 0.2
    values[m] = np.round(values[m])
    root_values = (values + rng.normal(0, 0.5, T)).astype(np.float32)
    to_play, action_mask = [], []
    for n in range(N):       # _preprocess_to_play_and_action_mask (lzero/mcts/buffer/game_buffer.py:480-522)
        tp = list(to_play_segment[n][pos[n]:pos[n] + K1])
        to_play += tp + [-1] * (K1 - len(tp))
        am = [list(x) for x in action_mask_segment[n][pos[n]:pos[n] + K1]]
        action_mask += am + [list(np.ones(A, np.int8)) for _ in range(K1 - len(am))]
    noises = np.stack([rng.dirichlet([0.3] * A).astype(np.float32) for _ in range(T)])
    return dict(value_mask=value_mask, pos=pos, rewards_list=rewards_list, game_segment_lens=lens, td_steps_list=td_steps_list,
                to_play_segment=to_play_segment, env_type="board_games" if two else "not_board_games", values=values,
                root_values=root_values, action_mask=np.asarray(action_mask, np.uint8), to_play=np.asarray(to_play, np.int32),
                noises=noises)
