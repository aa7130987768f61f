"""Host side of the ReZero reanalyze sweep, without a GPU.

  - the row <-> (segment, position) mapping and the backward order the device sweep uses (search it takes row segment * L +
    L - 1 - it) against compute_all_filters (game_buffer_rezero_mz.py:19-26, restated), and the reference's reassembly of the
    per-search results (reverse, then zip per segment) against the [N, L] layout of the outputs;
  - the buffer write-back and the ReZero statistics against the reference's assembly on synthetic distributions;
  - the refusals (length < 1, wrong tree / model pairs), which happen before any device is touched;
  - k_rezero_handoff / k_rezero_targets: no spills, no local memory, and rezero.cu compiled without fp32 contraction.
"""
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from conftest import ROOT


def compute_all_filters(data, num_unroll_steps):
    """game_buffer_rezero_mz.py:19-26"""
    data_by_iter = []
    for it in range(num_unroll_steps + 1):
        iter_data = [x for i, x in enumerate(data)
                     if (i + 1) % (num_unroll_steps + 1) == ((num_unroll_steps + 1 - it) % (num_unroll_steps + 1))]
        data_by_iter.append(iter_data)
    return data_by_iter


@pytest.mark.parametrize("N, L", [(1, 1), (7, 1), (1, 2), (7, 2), (3, 6), (256, 5)])
def test_rows_and_backward_order_match_compute_all_filters(N, L):
    by_iter = compute_all_filters(list(range(N * L)), L - 1)
    assert by_iter == [[n * L + L - 1 - it for n in range(N)] for it in range(L)]
    # the reference's reassembly: temp_*.reverse(); extend(column for column in zip(*temp)) -> row order
    temp = [[("it", it, n) for n in range(N)] for it in range(L)]
    temp.reverse()
    flat = []
    [flat.extend(column) for column in zip(*temp)]
    assert flat == [("it", L - 1 - p, n) for n in range(N) for p in range(L)]      # row n * L + p <- search L - 1 - p


def _reference_assembly(dists, values, policy_mask, legal, pos, L, A, scatter):
    """game_buffer_rezero_mz.py:361-392 on per-row distributions (legal order) and values"""
    child_visits, root_values, targets = [dict() for _ in pos], [dict() for _ in pos], []
    policy_index = 0
    for state_index, child_visit, root_value in zip(pos, child_visits, root_values):
        target_policies = []
        for current_index in range(state_index, state_index + L):
            distributions = dists[policy_index]
            if policy_mask[policy_index] == 0:
                target_policies.append([0 for _ in range(A)])
            else:
                sim_num = sum(distributions)
                child_visit[current_index] = [v / sim_num for v in distributions]
                root_value[current_index] = values[policy_index]
                policy = [v / sim_num for v in distributions]
                if scatter:
                    tmp = [0 for _ in range(A)]
                    for index, legal_action in enumerate(legal[policy_index]):
                        tmp[legal_action] = policy[index]
                    policy = tmp
                target_policies.append(policy)
            policy_index += 1
        targets.append(target_policies)
    return np.array(targets), child_visits, root_values


@pytest.mark.parametrize("scatter", [False, True])
def test_write_back_and_targets_match_reference_assembly(scatter):
    from lightzero_b200.reanalyze import rezero_write_back
    rng = np.random.default_rng(3)
    N, L, A, S = 5, 4, 7, 50
    rows = N * L
    mask = np.ones((rows, A), np.uint8)
    if scatter:
        mask = (rng.random((rows, A)) < 0.5).astype(np.uint8)
        mask[np.arange(rows), rng.integers(0, A, rows)] = 1
    legal = [np.nonzero(m)[0].tolist() for m in mask]
    dists = [rng.multinomial(S, np.ones(len(l)) / len(l)).tolist() for l in legal]
    values = rng.standard_normal(rows).astype(np.float32)
    pm = (rng.random(rows) < 0.8).astype(np.uint8)
    pos = rng.integers(0, 100, N).tolist()
    exp_targets, exp_cv, exp_rv = _reference_assembly(dists, values.tolist(), pm, legal, pos, L, A, scatter)
    # what k_rezero_targets writes: visit / sum in float64 by legal position or action id, zeros where policy_mask == 0
    visits = np.zeros((N, L, A))
    targets = np.zeros((N, L, A))
    for i, (d, l) in enumerate(zip(dists, legal)):
        n, p = divmod(i, L)
        v = np.asarray(d, np.float64) / float(sum(d))
        visits[n, p, :len(d)] = v
        if pm[i]:
            targets[n, p, l if scatter else np.arange(len(d))] = v
    assert np.array_equal(targets.view(np.uint64), np.asarray(exp_targets, np.float64).view(np.uint64))
    cv, rv = [dict() for _ in pos], [dict() for _ in pos]
    rezero_write_back(cv, rv, pos, L, pm, mask, visits, values.reshape(N, L))
    assert cv == exp_cv and rv == exp_rv


def test_reuse_stats_match_reference_accumulation():
    from lightzero_b200.reanalyze import rezero_reuse_stats
    rng = np.random.default_rng(4)
    S = 13
    counts = rng.integers(0, 64, (5, S)).astype(np.int32)
    temp_length, temp_infer = 0, 0
    for c in counts:                    # search_with_reuse returns (length, infer_sum / num_simulations), mcts_ctree.py:464-467
        temp_length += int(c[-1])
        temp_infer += int(c.sum()) / S
    assert rezero_reuse_stats(counts, S) == (temp_length / 5, temp_infer / 5)
    assert rezero_reuse_stats(np.zeros((0, S), np.int32), S) == (0, 0.0)


def test_refusals():
    import lightzero_b200 as lzb
    from lightzero_b200.reanalyze import compute_target_policy_reanalyzed_rezero as sweep
    args = (np.zeros((2, 4), np.float32), np.ones((2, 2), np.uint8), [-1, -1], [0, -2], [1, 1], [0])
    for length in (0, -1):
        with pytest.raises(ValueError):
            sweep(object(), lzb.MuZeroMCTSCtree(), *args, length)
    for mcts in (lzb.MuZeroMCTSCtree(), lzb.EfficientZeroMCTSCtree(), lzb.GumbelMuZeroMCTSCtree(), object()):
        with pytest.raises(TypeError):
            sweep(object(), mcts, *args, 2)


# ---- kernel resources (nvcc, no GPU) ----
@pytest.fixture(scope="module")
def compiled():
    if shutil.which("nvcc") is None or shutil.which("cuobjdump") is None:
        pytest.skip("nvcc / cuobjdump not on PATH")
    from lightzero_b200 import _build
    flags = dict(_build.UNITS)["rezero.cu"]
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        for name, extra in (("build", flags), ("fmad", ["-fmad=true"])):
            obj = os.path.join(tmp, name + ".o")
            cmd = ["nvcc"] + _build.ARCH + _build.COMMON + extra + ["-Xptxas", "-v", "-c",
                                                                   os.path.join(ROOT, "lightzero_b200", "csrc", "rezero.cu"), "-o", obj]
            p = subprocess.run(cmd, capture_output=True, text=True)
            assert p.returncode == 0, p.stderr[-4000:]
            sass = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
            out[name] = (p.stdout + p.stderr, sass)
    return flags, out


def _functions(sass):
    """kernel name -> its SASS"""
    parts = re.split(r"\n\s*Function : ", sass)
    return {re.search(r"(k_rezero_(?:handoff|targets))", p.split("\n", 1)[0]).group(1): p for p in parts[1:] if "k_rezero_" in p.split("\n", 1)[0]}


def test_rezero_kernels_neither_spill_nor_use_local_memory(compiled):
    _, out = compiled
    log, sass = out["build"]
    for line in log.splitlines():
        if "spill" in line:
            assert "0 bytes spill stores, 0 bytes spill loads" in line, line
    funcs = _functions(sass)
    assert set(funcs) == {"k_rezero_handoff", "k_rezero_targets"}
    for name, body in funcs.items():
        assert not re.search(r"\b(LDL|STL)\b", body), name


def test_rezero_unit_has_no_fp32_contraction(compiled):
    """rezero.cu is built with -fmad=false, and neither kernel has an fp32 multiply-add that contraction could have made: a build
    that allows contraction has exactly the same FFMA count in each kernel (the FFMA present are the exactly rounded division
    sequences of __fdiv_rn / __ddiv_rn)."""
    flags, out = compiled
    assert "-fmad=false" in flags
    built, fmad = _functions(out["build"][1]), _functions(out["fmad"][1])
    for name in ("k_rezero_handoff", "k_rezero_targets"):
        assert built[name].count("FFMA") == fmad[name].count("FFMA"), name
