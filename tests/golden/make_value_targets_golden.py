"""Writes tests/golden/value_targets.npz: what the reference's own ``MuZeroGameBuffer._compute_target_reward_value``
(lzero/mcts/buffer/game_buffer_muzero.py:467-575) and ``EfficientZeroGameBuffer._compute_target_reward_value``
(game_buffer_efficientzero.py:167-323) return, on the CPU, for every case of tests/value_targets_cases.py.

The two methods, ``_scalar_reward``, ``_preprocess_to_play_and_action_mask`` and the helpers they call (prepare_observation,
to_detach_cpu_numpy, concat_output, concat_output_value) are compiled out of the reference's source files with ``ast`` into one
namespace, so the buffer modules (and DI-engine, which they import) are never imported.  The namespace supplies:
  - a stand-in model whose initial_inference returns the case's recorded fp32 value scalars for the rows it is given (the
    observations are row numbers), with ``inverse_scalar_transform`` the identity on them: the targets bootstrap from exactly
    those scalars;
  - a stand-in MCTS (EfficientZero use_root_value) whose roots return the case's recorded root values from get_values();
  - the buffer's config (EasyDict-like attribute dict).
For MuZero with use_root_value=True the generator records that the reference raises (a broadcast ValueError).

Run where the reference sources are (LZ_REFERENCE, default /root/reference):   python tests/golden/make_value_targets_golden.py
"""
import ast
import os
import sys
from typing import Any, List, Optional, Tuple, Union

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
from value_targets_cases import CASES, MZ_ROOT_FAILURE, make_context, seed_of  # noqa: E402

OUT = os.path.join(HERE, "value_targets.npz")


class AttrDict(dict):
    __getattr__ = dict.__getitem__


def compile_functions(ref, relpath, names, ns, cls=None):
    """Executes the named top-level functions (or methods of class cls) of ref/relpath in ns."""
    tree = ast.parse(open(os.path.join(ref, relpath)).read())
    body = tree.body
    if cls is not None:
        body = next(n for n in tree.body if isinstance(n, ast.ClassDef) and n.name == cls).body
    fns = [n for n in body if isinstance(n, ast.FunctionDef) and n.name in names]
    assert {f.name for f in fns} == set(names), (relpath, names)
    for f in fns:
        f.decorator_list = []
    exec(compile(ast.Module(body=fns, type_ignores=[]), os.path.join(ref, relpath), "exec"), ns)
    return {f.name: ns[f.name] for f in fns}


class StubOutput:
    def __init__(self, rows, values, A):
        B = len(rows)
        self.value = torch.from_numpy(values[rows].reshape(B, 1))
        self.policy_logits = torch.zeros(B, A)
        self.latent_state = torch.zeros(B, 2)
        self.reward = [0.0] * B
        self.value_prefix = torch.zeros(B, 1)
        self.reward_hidden_state = (torch.zeros(1, B, 3), torch.zeros(1, B, 3))


class StubModel:
    training = False

    def __init__(self, values, A):
        self.values, self.A = values, A

    def initial_inference(self, obs, **_):
        return StubOutput(obs.reshape(obs.shape[0], -1)[:, 0].numpy().astype(np.int64), self.values, self.A)


class StubRoots:
    root_values = None

    def __init__(self, n, legal):
        self.n = n

    def prepare(self, *a):
        pass

    def prepare_no_noise(self, *a):
        pass

    def get_values(self):
        return [float(v) for v in StubRoots.root_values]


class StubMCTS:
    def __init__(self, cfg):
        pass

    @classmethod
    def roots(cls, n, legal):
        return StubRoots(n, legal)

    def search(self, *a, **k):
        pass


def to_list(x):
    return x.tolist() if isinstance(x, np.ndarray) else [to_list(v) for v in x] if isinstance(x, (list, tuple)) else x


def load(ref):
    ns = dict(np=np, torch=torch, Any=Any, List=List, Tuple=Tuple, Union=Union, Optional=Optional, to_list=to_list,
              inverse_scalar_transform=lambda v, support: v, MCTSCtree=StubMCTS, MCTSPtree=StubMCTS)
    compile_functions(ref, "lzero/mcts/utils.py", ["prepare_observation"], ns)
    compile_functions(ref, "lzero/policy/utils.py", ["to_detach_cpu_numpy", "concat_output", "concat_output_value"], ns)
    pre = compile_functions(ref, "lzero/mcts/buffer/game_buffer.py", ["_preprocess_to_play_and_action_mask"], dict(ns),
                            cls="GameBuffer")
    mz = compile_functions(ref, "lzero/mcts/buffer/game_buffer_muzero.py", ["_compute_target_reward_value", "_scalar_reward"],
                           dict(ns), cls="MuZeroGameBuffer")
    ez = compile_functions(ref, "lzero/mcts/buffer/game_buffer_efficientzero.py", ["_compute_target_reward_value"], dict(ns),
                           cls="EfficientZeroGameBuffer")
    MZ = type("MZBuffer", (), dict(mz, **pre))
    EZ = type("EZBuffer", (), dict(ez, _scalar_reward=mz["_scalar_reward"], **pre))
    return MZ, EZ


def run_case(MZ, EZ, case, ctx, A=6):
    T = case["N"] * case["K1"]
    cfg = AttrDict(num_unroll_steps=case["K1"] - 1, discount_factor=case["discount"], env_type=ctx["env_type"],
                   mini_infer_size=5 if T > 5 else 2, use_root_value=bool(case.get("root")), device="cpu",
                   lstm_horizon_len=case.get("H", 5), reanalyze_noise=True, root_noise_weight=0.25, root_dirichlet_alpha=0.3,
                   mcts_ctree=True, model=AttrDict(model_type="mlp", action_space_size=A, continuous_action_space=False))
    buf = (EZ if case["kind"] == "ez" else MZ)()
    buf._cfg, buf.value_support, buf.task_id = cfg, None, None
    obs = np.arange(T, dtype=np.float32).reshape(T, 1, 1)      # [B, S, O]: one stacked frame of one feature, the row number
    StubRoots.root_values = ctx["root_values"]
    model = StubModel(ctx["values"], A)
    if case["kind"] == "ez":
        context = [obs, ctx["value_mask"], ctx["pos"], ctx["rewards_list"], ctx["game_segment_lens"], ctx["td_steps_list"],
                   [None] * case["N"], ctx["to_play_segment"]]
        # the action masks the root search would see: the stand-in segments' masks through _preprocess_to_play_and_action_mask
        context[6] = [np.ones((len(t), A), np.int8) for t in ctx["to_play_segment"]]
    else:
        context = [obs, ctx["value_mask"], ctx["pos"], ctx["rewards_list"], [], ctx["game_segment_lens"], ctx["td_steps_list"],
                   [None] * case["N"], ctx["to_play_segment"]]
    r, v = buf._compute_target_reward_value(context, model)
    flat = np.vectorize(lambda x: float(np.asarray(x).reshape(-1)[0]), otypes=[np.float64])
    if r.dtype == object and r.ndim == 3:      # (n, 1) rewards in an object array: one more axis
        r, v = r[..., 0], v[..., 0] if v.ndim == 3 else v
    return flat(r).astype(np.float64), flat(v).astype(np.float64)


def pack(name, case, ctx, r, v):
    d = {}
    d["kind"] = np.array(case["kind"])
    for k in ("N", "K1", "td", "players"):
        d[k] = np.int64(case[k])
    d["discount"] = np.float64(case["discount"])
    d["H"] = np.int64(case.get("H", 5))
    d["root"] = np.int64(bool(case.get("root")))
    d["rewards_kind"] = np.array(case["rewards"])
    d["env_type"] = np.array(ctx["env_type"])
    d["pos"] = np.asarray(ctx["pos"], np.int64)
    d["game_segment_lens"] = np.asarray(ctx["game_segment_lens"], np.int64)
    d["reward_lens"] = np.asarray([len(x) for x in ctx["rewards_list"]], np.int64)
    d["rewards_flat"] = np.concatenate([x.reshape(-1) for x in ctx["rewards_list"]])
    d["to_play_lens"] = np.asarray([len(x) for x in ctx["to_play_segment"]], np.int64)
    d["to_play_flat"] = np.concatenate(ctx["to_play_segment"])
    d["td_steps"] = np.asarray(ctx["td_steps_list"], np.int32)
    d["value_mask"] = np.asarray(ctx["value_mask"], np.int64)
    d["values"] = ctx["values"]
    d["root_values"] = ctx["root_values"]
    d["exp_rewards"] = r
    d["exp_values"] = v
    return {f"{name}/{k}": x for k, x in d.items()}


def main(ref):
    MZ, EZ = load(ref)
    out = {}
    for name, case in CASES.items():
        ctx = make_context(case, seed_of(name))
        r, v = run_case(MZ, EZ, case, ctx)
        out.update(pack(name, case, ctx, r, v))
        print(f"{name}: rewards {r.shape}, values {v.shape}, -0.0 values {int(np.sum(np.signbit(v) & (v == 0)))}")
    ctx = make_context(MZ_ROOT_FAILURE, seed_of("mz_root_failure"))
    try:
        run_case(MZ, EZ, MZ_ROOT_FAILURE, ctx)
        msg = ""
    except ValueError as e:
        msg = str(e)
    assert "broadcast" in msg, msg
    print("mz use_root_value:", msg)
    out["mz_root_failure/message"] = np.array(msg)
    np.savez_compressed(OUT, **out)
    print("wrote", OUT)


if __name__ == "__main__":
    main(os.environ.get("LZ_REFERENCE", "/root/reference"))
