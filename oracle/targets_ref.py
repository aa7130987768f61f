"""The replay buffer's reward and value targets, restated for the tests.  TEST INFRASTRUCTURE ONLY.

``reward_value_targets`` computes what ``MuZeroGameBuffer._compute_target_reward_value`` (lzero/mcts/buffer/
game_buffer_muzero.py:467-575) and ``EfficientZeroGameBuffer._compute_target_reward_value`` (game_buffer_efficientzero.py:167-323)
return for given fp32 bootstrap values (the network's value scalars, or EfficientZero's searched root values).  It keeps the
operand types the reference's arithmetic has, because they decide the rounding:
  - bootstrap: (float32 value -> float64) * discount ** td (negated for odd td in two-player board games) * value_mask, float64;
  - window terms reward * discount ** i: a float32 product with the Python-float power rounded to float32 for float32 rewards,
    float64 otherwise; the first += makes the Python-float accumulator a float32 one (NEP 50), after which every add is float32;
  - the two-player sign compares to_play_list[base_index] with to_play_list[i], i the offset into the window;
  - EfficientZero: horizon_id counts rows across segments; at every lstm_horizon_len-th row, after that row's window sum, the
    prefix restarts at 0.0 and base_index moves to the row; (n, 1) rewards make the prefix an array that later rows add to in
    place, so every row appended since the restart reads the last prefix.
Returns float64 arrays [N, K + 1]: the reference's elements as Python floats (its object arrays flattened element by element).
"""
import numpy as np


def reward_value_targets(values, value_mask, pos_in_game_segment_list, rewards_list, game_segment_lens, td_steps_list,
                         to_play_segment, num_unroll_steps=5, discount_factor=0.997, env_type="not_board_games",
                         efficientzero=False, lstm_horizon_len=5):
    K1 = num_unroll_steps + 1
    N = len(pos_in_game_segment_list)
    T = N * K1
    d = discount_factor
    two = env_type == "board_games" and to_play_segment[0][0] in [1, 2]
    disc = np.empty(T, np.float64)
    for j in range(T):
        p = d ** td_steps_list[j]
        disc[j] = -p if two and int(td_steps_list[j]) % 2 else p
    if not two:
        disc = np.array([d] * T) ** np.asarray(td_steps_list)
    boot = (np.asarray(values, np.float32).reshape(-1) * disc * np.array(value_mask)).tolist()

    rewards_out = np.zeros((N, K1), np.float64)
    values_out = np.zeros((N, K1), np.float64)

    def scalar(x):
        return float(np.asarray(x).reshape(-1)[0])

    row = 0
    for n in range(N):
        rl, tp, start = rewards_list[n], to_play_segment[n], pos_in_game_segment_list[n]
        base = start
        prefix = 0.0
        appended = []          # (row, prefix object) of this segment, read once the segment is done
        for k in range(K1):
            cur = start + k
            acc = boot[row]
            for i, r in enumerate(rl[cur:cur + td_steps_list[row]]):
                term = r * d ** i
                if two and tp[base] != tp[i]:
                    term = -r * d ** i
                acc = acc + term if not isinstance(acc, np.ndarray) else _iadd(acc, term)
            if efficientzero:
                if row % lstm_horizon_len == 0:
                    prefix = 0.0
                    base = cur
                if cur < game_segment_lens[n]:
                    values_out[n, k] = scalar(acc)
                    prefix = _iadd(prefix, rl[cur]) if isinstance(prefix, np.ndarray) else prefix + rl[cur]
                else:
                    values_out[n, k] = 0.0
                appended.append((k, prefix))
            else:
                values_out[n, k] = scalar(acc)
                rewards_out[n, k] = scalar(rl[cur]) if cur < len(rl) else 0.0
            row += 1
        for k, obj in appended:
            rewards_out[n, k] = scalar(obj)
    return rewards_out, values_out


def _iadd(a, b):
    a += b          # in place: every list entry holding this array sees the sum
    return a
