"""The replay buffer's reward / value targets without a GPU.

- oracle/targets_ref.py reproduces, bit for bit (float64 bit patterns, so -0.0 counts), what the reference's own
  _compute_target_reward_value returned for every case of tests/golden/value_targets.npz (make_value_targets_golden.py).
- reanalyze.pack_value_targets packs those contexts into the tables of lz_value_tables; k_value_targets restated over the
  packed tables (one segment at a time, its float32 / float64 operations spelled out as in csrc/targets.cu) gives the same bits.
- The refusals of compute_target_reward_value.
- k_value_targets neither spills nor uses local memory, and targets.cu has no FFMA / DFMA contraction.
"""
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from conftest import GOLDEN_DIR, ROOT
from oracle.targets_ref import reward_value_targets
from value_targets_cases import CASES, MZ_ROOT_FAILURE, make_context, seed_of

FIXTURE = os.path.join(GOLDEN_DIR, "value_targets.npz")


def load_case(name):
    z = np.load(FIXTURE)
    g = {k.split("/", 1)[1]: z[k] for k in z.files if k.startswith(name + "/")}
    dtype = np.float64 if str(g["rewards_kind"]).startswith("f64") else np.float32
    column = str(g["rewards_kind"]).endswith("x1")
    rl = np.split(g["rewards_flat"].astype(dtype), np.cumsum(g["reward_lens"])[:-1])
    rl = [r.reshape(-1, 1) if column else r for r in rl]
    tps = np.split(g["to_play_flat"], np.cumsum(g["to_play_lens"])[:-1])
    ctx = dict(value_mask=g["value_mask"].tolist(), pos=g["pos"].tolist(), rewards_list=rl,
               game_segment_lens=g["game_segment_lens"].tolist(), td_steps_list=list(g["td_steps"]), to_play_segment=tps,
               env_type=str(g["env_type"]))
    cfg = dict(num_unroll_steps=int(g["K1"]) - 1, discount_factor=float(g["discount"]), efficientzero=str(g["kind"]) == "ez",
               lstm_horizon_len=int(g["H"]))
    values = g["root_values"] if int(g["root"]) else g["values"]
    return ctx, cfg, values, g["exp_rewards"], g["exp_values"]


def context_args(ctx):
    return (ctx["value_mask"], ctx["pos"], ctx["rewards_list"], ctx["game_segment_lens"], ctx["td_steps_list"],
            ctx["to_play_segment"])


def same_bits(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return a.shape == b.shape and np.array_equal(a.view(np.uint64), b.view(np.uint64))


def test_fixture_covers_the_case_grid():
    z = np.load(FIXTURE)
    assert {k.split("/")[0] for k in z.files} == set(CASES) | {"mz_root_failure"}
    assert "broadcast" in str(z["mz_root_failure/message"])
    # the generator draws its contexts from the shared case grid
    ctx, _, values, _, _ = load_case("mz_2p_f32_n64_k6")
    again = make_context(CASES["mz_2p_f32_n64_k6"], seed_of("mz_2p_f32_n64_k6"))
    assert np.array_equal(values, again["values"]) and ctx["pos"] == again["pos"]
    seen = {(c["kind"], c["rewards"], c["players"], c["td"], c["discount"], c.get("H"), c["N"], c["K1"]) for c in CASES.values()}
    assert {s[1] for s in seen} == {"f32", "f64", "f32x1", "f64x1"} and {s[3] for s in seen} == {1, 5, 9}
    assert {s[4] for s in seen} == {0.997, 1.0} and {s[5] for s in seen} >= {1, 5}
    assert {s[6] for s in seen} == {1, 7, 64} and {s[7] for s in seen} == {1, 6}


@pytest.mark.parametrize("name", sorted(CASES))
def test_restatement_matches_reference(name):
    ctx, cfg, values, exp_r, exp_v = load_case(name)
    r, v = reward_value_targets(values, *context_args(ctx), env_type=ctx["env_type"], **cfg)
    assert same_bits(r, exp_r), "rewards / value prefixes differ"
    assert same_bits(v, exp_v), "value targets differ"


def restate_kernel(f, t, values):
    """k_value_targets (csrc/targets.cu) over the packed tables, one segment at a time"""
    N, K1, P = f["N"], f["K1"], f["P"]
    f32 = f["fp32"]

    def add(acc, term):
        return float(np.float32(acc) + np.float32(term)) if f32 else acc + term
    rew, val = np.zeros((N, K1)), np.zeros((N, K1))
    for n in range(N):
        rw, rlen = t["rewards"][n], int(t["rlen"][n])
        tp = t["to_play"][n] if f["two_player"] else None
        prefix, live, chunk0, base = 0.0, False, 0, 0
        for k in range(K1):
            r = n * K1 + k
            acc = float(np.float64(np.float32(values[r])) * t["bootstrap"][r] * t["value_mask"][r])
            end = min(k + int(t["td"][r]), rlen)
            for i in range(max(0, end - k)):
                x = -rw[k + i] if tp is not None and tp[i] != tp[P + base] else rw[k + i]
                term = float(np.float32(x) * np.float32(t["powers"][i])) if f32 else x * t["powers"][i]
                acc = add(acc, term)
            if not f["value_prefix"]:
                val[n, k], rew[n, k] = acc, (rw[k] if k < rlen else 0.0)
                continue
            if r % f["horizon"] == 0:
                if f["alias_prefix"] and live:
                    rew[n, chunk0:k] = prefix
                prefix, live, base = 0.0, False, k
            if k < t["seglen"][n]:
                val[n, k] = acc
                prefix = add(prefix, rw[k])
                if not live:
                    live, chunk0 = True, k
            else:
                val[n, k] = 0.0
            rew[n, k] = prefix
        if f["alias_prefix"] and live:
            rew[n, chunk0:] = prefix
    return rew, val


@pytest.mark.parametrize("name", sorted(CASES))
def test_packed_tables_give_reference_targets(name):
    from lightzero_b200.reanalyze import pack_value_targets
    ctx, cfg, values, exp_r, exp_v = load_case(name)
    f, t = pack_value_targets(*context_args(ctx), env_type=ctx["env_type"], **cfg)
    assert f["W"] == f["K1"] - 1 + f["P"] and t["rewards"].shape == (f["N"], f["W"])
    assert t["bootstrap"].dtype == np.float64 and t["powers"].dtype == np.float64 and t["td"].dtype == np.int32
    r, v = restate_kernel(f, t, values)
    assert same_bits(r, exp_r), "rewards / value prefixes differ"
    assert same_bits(v, exp_v), "value targets differ"


def test_pack_layout():
    from lightzero_b200.reanalyze import pack_value_targets
    rl = [np.array([1, 2, 3, 4], np.float32), np.array([5, 6], np.float32)]
    f, t = pack_value_targets([1, 0, 0, 0], [1, 1], rl, [4, 2], [np.int32(2)] * 4, [np.full(4, -1), np.full(2, -1)],
                              num_unroll_steps=1, discount_factor=0.5)
    assert (f["N"], f["K1"], f["P"], f["W"], f["fp32"], f["two_player"]) == (2, 2, 2, 3, 1, 0)
    assert t["rewards"].tolist() == [[2, 3, 4], [6, 0, 0]] and t["rlen"].tolist() == [3, 1]
    assert t["powers"].tolist() == [1.0, 0.5] and t["bootstrap"].tolist() == [0.25] * 4 and t["to_play"] is None


def test_refusals():
    from lightzero_b200.reanalyze import compute_target_reward_value as crv
    ctx = make_context(CASES["mz_f32_n7_k6"], 1)
    obs = np.zeros((42, 4), np.float32)
    args = (obs, ctx["value_mask"], ctx["pos"], ctx["rewards_list"], ctx["game_segment_lens"], ctx["td_steps_list"],
            ctx["to_play_segment"])
    with pytest.raises(ValueError, match="broadcast"):                 # MuZeroGameBuffer's use_root_value fails in the reference
        crv(object(), *args, use_root_value=True)
    with pytest.raises(TypeError):                                     # not a CUDA model
        crv(object(), *args)
    with pytest.raises(ValueError):                                    # no segments
        crv(object(), np.zeros((0, 4), np.float32), [], [], [], [], [], [])
    with pytest.raises(ValueError):                                    # 6 rows per segment, 5 value_mask entries per segment
        crv(object(), *args[:1], ctx["value_mask"][:-7], *args[2:])
    with pytest.raises(ValueError):                                    # one reward list missing
        crv(object(), *args[:3], ctx["rewards_list"][:-1], *args[4:])
    with pytest.raises(ValueError):                                    # value_obs rows
        crv(object(), obs[:-1], *args[1:])
    with pytest.raises(TypeError):                                     # integer rewards
        crv(object(), *args[:3], [r.astype(np.int64) for r in ctx["rewards_list"]], *args[4:])
    with pytest.raises(TypeError):                                     # float16 rewards
        crv(object(), *args[:3], [r.astype(np.float16) for r in ctx["rewards_list"]], *args[4:])
    with pytest.raises(TypeError):                                     # float32 and float64 segments mixed
        crv(object(), *args[:3], [r.astype(np.float64) if i % 2 else r for i, r in enumerate(ctx["rewards_list"])], *args[4:])
    with pytest.raises(ValueError):                                    # EfficientZero: a reward list shorter than its segment
        crv(object(), *args[:3], [r[:1] for r in ctx["rewards_list"]], [100] * 7, *args[5:], efficientzero=True)
    two = make_context(CASES["mz_2p_f32_n64_k6"], 2)
    with pytest.raises(ValueError):                                    # two players: a to_play list shorter than the window reads
        crv(object(), np.zeros((384, 4), np.float32), two["value_mask"], two["pos"], two["rewards_list"],
            two["game_segment_lens"], two["td_steps_list"], [t[:1] for t in two["to_play_segment"]], env_type="board_games")


def test_mz_root_value_failure_is_the_references():
    """The generator ran MuZeroGameBuffer._compute_target_reward_value with use_root_value=True: it raised the broadcast error
    that compute_target_reward_value refuses the call for"""
    z = np.load(FIXTURE)
    T = MZ_ROOT_FAILURE["N"] * MZ_ROOT_FAILURE["K1"]
    assert f"(0,) ({T},)" in str(z["mz_root_failure/message"])


# ---- kernel resources (nvcc, no GPU) ----
@pytest.fixture(scope="module")
def compiled():
    if shutil.which("nvcc") is None or shutil.which("cuobjdump") is None:
        pytest.skip("nvcc / cuobjdump not on PATH")
    from lightzero_b200 import _build
    flags = dict(_build.UNITS)["targets.cu"]
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        for name, extra in (("build", flags), ("fmad", ["-fmad=true"])):
            obj = os.path.join(tmp, name + ".o")
            cmd = ["nvcc"] + _build.ARCH + _build.COMMON + extra + ["-Xptxas", "-v", "-c",
                                                                   os.path.join(ROOT, "lightzero_b200", "csrc", "targets.cu"), "-o", obj]
            p = subprocess.run(cmd, capture_output=True, text=True)
            assert p.returncode == 0, p.stderr[-4000:]
            sass = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
            out[name] = (p.stdout + p.stderr, sass)
    return flags, out


def _kernel(sass):
    parts = re.split(r"\n\s*Function : ", sass)
    bodies = [p for p in parts[1:] if "k_value_targets" in p.split("\n", 1)[0]]
    assert len(bodies) == 1
    return bodies[0]


def test_value_targets_kernel_neither_spills_nor_uses_local_memory(compiled):
    _, out = compiled
    log, sass = out["build"]
    for line in log.splitlines():
        if "spill" in line:
            assert "0 bytes spill stores, 0 bytes spill loads" in line, line
    assert not re.search(r"\b(LDL|STL)\b", _kernel(sass))


def test_targets_unit_has_no_contraction(compiled):
    """targets.cu is built with -fmad=false and k_value_targets has float32 and float64 products and sums, none fused; every
    operation is an explicit __f*_rn / __d*_rn, so a build that allows contraction has no fused one either"""
    flags, out = compiled
    assert "-fmad=false" in flags
    built, fmad = _kernel(out["build"][1]), _kernel(out["fmad"][1])
    assert re.search(r"\bDMUL\b", built) and re.search(r"\bDADD\b", built)
    assert re.search(r"\bFMUL\b", built) and re.search(r"\bFADD\b", built)
    assert not re.search(r"\b(DFMA|FFMA)\b", built)
    assert not re.search(r"\b(DFMA|FFMA)\b", fmad)
