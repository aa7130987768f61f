"""CPU tests of the Stochastic MuZero pieces that need no GPU:
- the chance draw: a Python restatement of std::mt19937 + generate_canonical<double, 53> + std::discrete_distribution
  (lightzero_b200.stochastic_mz_tree.chance_uniform and the lower_bound below, which csrc/tree.cuh's chance_outcome
  computes on the device) picks the outcome the compiled reference tree picks, with std::random_device pinned by
  oracle/random_device_shim.cc, for many (seed, priors) pairs;
- the model and config refusals of StochasticMuZeroModelMLP and lz_model_create_mlp_stochastic, and
  StochasticMuZeroMCTSCtree's refusal of search_with_reuse;
- the kernels a stochastic search runs (every k_mez_tc instantiation and the MuZero k_tree_step<false, false>, which holds the
  chance draw) use no local memory and do not spill."""
import os
import re
import shutil
import subprocess
import tempfile

import numpy as np
import pytest

from conftest import ROOT
from lightzero_b200.stochastic_mz_tree import chance_uniform

CSRC = os.path.join(ROOT, "lightzero_b200", "csrc")


def discrete_draw(priors, u):
    """std::discrete_distribution<>(priors) at the uniform u in libstdc++ (param_type::_M_initialize, operator())"""
    p = [float(np.float32(x)) for x in priors]
    if len(p) < 2:
        return 0
    s = 0.0
    for x in p:
        s += x
    cp = [0.0] * len(p)
    acc = 0.0
    for k, x in enumerate(p):
        acc += x / s
        cp[k] = acc
    cp[-1] = 1.0
    return next(k for k, c in enumerate(cp) if not c < u)


def test_mt19937_outputs():
    # std::mt19937's 10000th output from the default seed 5489 is 4123659995 (C++11 [rand.predef]); the restated
    # generate_canonical of the first two outputs follows from the first two
    from lightzero_b200.stochastic_mz_tree import _mt19937_first2
    assert _mt19937_first2(5489) == [3499211612, 581869302]
    g1, g2 = 3499211612, 581869302
    assert chance_uniform(5489) == (g1 + g2 * 2.0 ** 32) / 2.0 ** 64


@pytest.fixture(scope="module")
def oracle():
    from oracle import build_stoch_ref
    mod = build_stoch_ref.load()
    if mod is None:
        pytest.skip("compiled reference Stochastic MuZero tree not built (no reference sources)")
    return mod, build_stoch_ref.set_random_device


def oracle_outcome(mod, set_rd, seed, chance_logits):
    """the outcome the compiled reference picks at a chance node whose priors are softmax(chance_logits): a root with one
    legal action, its chance child expanded with those logits, then one descent through it"""
    set_rd(seed)
    r = mod.Roots(1, [[0]], len(chance_logits))
    r.prepare_no_noise([0.0], [[0.0]], [-1])
    mm = mod.MinMaxStatsList(1)
    mm.set_delta(0.01)
    res = mod.ResultsWrapper(1)
    mod.batch_traverse(r, 19652, 1.25, 0.997, mm, res, [-1])
    mod.batch_backpropagate(1, 0.997, [0.0], [0.0], [list(chance_logits)], mm, res, [-1], [True], [0])
    res = mod.ResultsWrapper(1)
    is_chance, _, _, last, _ = mod.batch_traverse(r, 19652, 1.25, 0.997, mm, res, [-1])
    assert is_chance == [False]
    return last[0]


def softmax32(x):
    """CNode::expand's priors (cnode.cpp:143-165): fp32 exp(l - max) / sequential fp32 sum"""
    x = np.asarray(x, np.float32)
    e = np.exp(x - x.max()).astype(np.float32)
    s = np.float32(0.0)
    for v in e:
        s = np.float32(s + v)
    return e / s


def test_chance_draw_matches_reference(oracle):
    mod, set_rd = oracle
    rng = np.random.default_rng(0)
    cases = 0
    for seed in list(range(40)) + [int(x) for x in rng.integers(0, 2 ** 32, 40)]:
        for C in (1, 2, 3, 5, 17):
            logits = (rng.standard_normal(C) * rng.choice([0.1, 1.0, 4.0])).astype(np.float32)
            got = oracle_outcome(mod, set_rd, seed, logits.tolist())
            assert got == discrete_draw(softmax32(logits), chance_uniform(seed)), (seed, C, logits)
            cases += 1
    assert cases == 400


def test_model_refusals():
    import lightzero_b200 as lzb
    base = dict(observation_shape=4, action_space_size=2, chance_space_size=3, latent_state_dim=128)
    for bad in (dict(categorical_distribution=False), dict(norm_type="LN"), dict(discrete_action_encoding_type="not_one_hot"),
                dict(state_norm=True), dict(reward_head_hidden_channels=[32, 32]), dict(value_head_hidden_channels=[]),
                dict(reward_support_range=(-10., 11., 1.))):
        with pytest.raises(NotImplementedError):
            lzb.StochasticMuZeroModelMLP(**base, **bad)


def test_search_with_reuse_refused():
    import lightzero_b200 as lzb
    with pytest.raises(NotImplementedError):
        lzb.StochasticMuZeroMCTSCtree(dict(num_simulations=5)).search_with_reuse(None, None, None, [-1], [0], [0.])


@pytest.mark.parametrize("field,value", [("latent_dim", 48), ("latent_dim", 16), ("latent_dim", 288), ("latent_dim", 512),
                                         ("chance_space_size", 0), ("chance_space_size", 609), ("action_space_size", 0),
                                         ("value_hidden", 33), ("policy_hidden", 0), ("obs_dim", 4097)])
def test_config_refusals(field, value):
    from lightzero_b200 import cabi
    lib = cabi.load()
    c = dict(obs_dim=4, action_space_size=2, chance_space_size=3, latent_dim=128, reward_hidden=32, value_hidden=32,
             policy_hidden=32, res_connection_in_dynamics=0, support_min=-300., support_max=301., support_step=1.)
    c[field] = value
    cfg = cabi.MlpStochasticConfig(*c.values())
    h = cabi.c_void_p()
    assert lib.lz_model_create_mlp_stochastic(cfg, h) < 0
    assert ("head hidden" if field.endswith("hidden") else field) in lib.lz_last_error().decode()


def _local_memory(obj):
    """kernel -> number of local-memory instructions (STL / LDL) in its SASS"""
    sass = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
    out, cur = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            out.setdefault(cur, 0)
        elif cur and re.search(r"\b(STL|LDL)\b", line):
            out[cur] += 1
    return out


def test_kernel_resources():
    if shutil.which("nvcc") is None or shutil.which("cuobjdump") is None:
        pytest.skip("nvcc / cuobjdump not on PATH")
    from lightzero_b200 import _build
    flags = dict(_build.UNITS)
    with tempfile.TemporaryDirectory() as tmp:
        logs, local = [], {}
        for unit, kernel in (("mlp_tc.cu", "k_mez_tc"), ("tree.cu", "k_tree_stepILb0ELb0E")):
            obj = os.path.join(tmp, unit.replace(".cu", ".o"))
            p = subprocess.run(["nvcc"] + _build.ARCH + _build.COMMON + flags[unit] + ["-Xptxas", "-v", "-c",
                               os.path.join(CSRC, unit), "-o", obj], capture_output=True, text=True)
            assert p.returncode == 0, p.stdout[-4000:] + p.stderr[-4000:]
            logs.append(p.stdout + p.stderr)
            local.update({k: v for k, v in _local_memory(obj).items() if kernel in k})
    log = "\n".join(logs)
    checked = 0
    for m in re.finditer(r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", log):
        if "k_mez_tc" in m.group(1) or "k_tree_stepILb0ELb0E" in m.group(1):
            assert m.group(3) == "0" and m.group(4) == "0", m.group(0)
            checked += 1
    assert checked == 9             # k_mez_tc<1 .. 8> and k_tree_step<false, false>
    assert len(local) == 9 and not any(local.values()), local
