"""End-to-end parity report at the north-star sizes (run on the GPU box, not a pytest): the CUDA pipeline vs the ORACLE pipeline
(compiled reference ctree + the PyTorch-CPU fp32 restatement of the reference model, deterministic=True) on the same seeded inputs:

  * fraction of roots whose visit-count distribution is identical, max |delta root value| over those roots and over all roots;
  * the oracle pipeline's recorded network outputs replayed through the CUDA trees (must reproduce the oracle bit for bit);
  * every diverging root classified: the first simulation at which the CUDA search and the oracle search pick a different
    (node, action), and the largest difference of the network outputs (value / reward scalars, policy logits) the two pipelines had
    fed that tree up to that point -- the data behind "PUCT is discontinuous: a 1e-6 difference in one prediction flips an arg-max".

Writes gpurun_out/parity_report.json and prints a markdown summary (copied to profiles/ by hand)."""
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import lightzero_b200 as lzb
from lightzero_b200 import mz_tree
from oracle.model_ref import MuZeroModelRef, emulate_trained_
from oracle.search_ref import SearchRef, collect_step_ref, load_tree_module
from oracle.tree_drive import assert_same, drive, from_recorder, recorded


class Recorder:
    """Wraps the CUDA model so that the step-wise device search records (latent index, action, outputs) per simulation."""

    def __init__(self, model, tree):
        self.model, self.tree, self.calls = model, tree, []

    def eval(self):
        return self

    def recurrent_inference(self, latent, action):
        out = self.model.recurrent_inference(latent, action, return_scalars=True)
        self.calls.append(dict(ix=self.tree.ix.cpu().numpy().copy(), action=action.cpu().numpy().copy(),
                               value=out.value_scalar.cpu().numpy().copy(), reward=out.reward_scalar.cpu().numpy().copy(),
                               policy=out.policy_logits.cpu().numpy().copy()))
        return out


def run(B, A, S, seed):
    torch.manual_seed(seed)
    ref = emulate_trained_(MuZeroModelRef((4, 84, 84), A), seed)
    cu = lzb.MuZeroModel(observation_shape=(4, 84, 84), action_space_size=A).load_state_dict(ref.state_dict())
    rng = np.random.default_rng(seed)
    obs = torch.rand(B, 4, 84, 84)
    mask = np.ones((B, A), np.uint8)
    legal = [list(range(A)) for _ in range(B)]
    noises = [rng.dirichlet([0.3] * A).astype(np.float32).tolist() for _ in range(B)]
    tree, kind = load_tree_module()
    rec = []
    t0 = time.time()
    exp = collect_step_ref(SearchRef(tree, num_simulations=S), ref, obs, mask, [-1] * B, noises=noises, recorder=rec)
    t_ref = time.time() - t0
    mcts = lzb.MuZeroMCTSCtree(dict(num_simulations=S, deterministic=True, discount_factor=0.997))
    out = cu.initial_inference(obs.cuda())
    # (1) the fused CUDA pipeline
    roots = mcts.roots(B, legal)
    roots.prepare(0.25, noises, [0.] * B, out.policy_logits, [-1] * B)
    mcts.search(roots, cu, out.latent_state, [-1] * B)
    got_d, got_v = roots.get_distributions(), np.asarray(roots.get_values(), np.float64)
    roots.clear()
    exp_v = np.asarray(exp["values"], np.float64)
    same = np.array([g == e for g, e in zip(got_d, exp["distributions"])])
    # (2) replay of the oracle's network outputs through the CUDA trees
    c = dict(B=B, A=A, S=S, legal=legal, root_logits=exp["policy_logits"], noises=noises, to_play=[-1] * B, **from_recorder(rec))
    trace, roots = drive(mz_tree, c, "mz", recorded(c))
    try:
        assert_same(trace, c)
        replay_ok = roots.get_distributions() == exp["distributions"] and bool(np.array_equal(
            np.asarray(roots.get_values(), np.float32).view(np.uint32), np.asarray(exp["values"], np.float32).view(np.uint32)))
    except AssertionError:
        replay_ok = False
    roots.clear()
    # (3) the same CUDA search step-wise with a recorder, to classify the diverging roots
    roots = mcts.roots(B, legal)
    roots.prepare(0.25, noises, [0.] * B, out.policy_logits, [-1] * B)
    roots._materialize(S, mcts._params())
    r = Recorder(cu, roots._tree)
    mcts.search(roots, r, out.latent_state, [-1] * B)
    step_d = roots.get_distributions()
    fused_equals_step = step_d == got_d
    first_div, dmax = [], []
    root_logit_diff = np.abs(out.policy_logits.cpu().numpy() - exp["policy_logits"]).max(1)
    for b in np.nonzero(~same)[0]:
        fd, dm = None, float(root_logit_diff[b])
        for s in range(S):
            c = r.calls[s]
            if int(c["ix"][b]) != int(rec[s]["ix"][b]) or int(c["action"][b]) != int(rec[s]["last_action"][b]):
                fd = s
                break
            dm = max(dm, abs(float(c["value"][b]) - rec[s]["value"][b]), abs(float(c["reward"][b]) - rec[s]["reward"][b]),
                     float(np.abs(c["policy"][b] - np.asarray(rec[s]["policy"][b])).max()))
        first_div.append(fd)
        dmax.append(dm)
    # network-output differences over ALL roots along the common prefix (first simulation: identical descents everywhere)
    c0 = r.calls[0]
    d_value0 = float(np.abs(c0["value"] - np.asarray(rec[0]["value"])).max())
    d_logit0 = float(np.abs(c0["policy"] - np.asarray(rec[0]["policy"])).max())
    return dict(B=B, A=A, S=S, seed=seed, tree_oracle=kind, oracle_seconds=round(t_ref, 1),
                identical_roots=int(same.sum()), identical_fraction=float(same.mean()),
                max_abs_dvalue_identical_roots=float(np.abs(got_v - exp_v)[same].max()) if same.any() else None,
                max_abs_dvalue_all_roots=float(np.abs(got_v - exp_v).max()),
                median_abs_dvalue_diverged_roots=float(np.median(np.abs(got_v - exp_v)[~same])) if (~same).any() else None,
                replay_of_oracle_outputs_bit_exact=bool(replay_ok), fused_equals_stepwise=bool(fused_equals_step),
                diverged=int((~same).sum()),
                first_divergent_simulation=dict(min=min([f for f in first_div if f is not None], default=None),
                                                median=float(np.median([f for f in first_div if f is not None])) if first_div else None,
                                                max=max([f for f in first_div if f is not None], default=None),
                                                none=sum(f is None for f in first_div)),
                max_network_output_diff_before_divergence=dict(max=max(dmax, default=None), median=float(np.median(dmax)) if dmax else None),
                first_simulation_max_abs_diff=dict(value_scalar=d_value0, policy_logits=d_logit0))


def main():
    cases = [(1024, 18, 50, 11), (128, 18, 200, 12)]
    if os.environ.get("PARITY_SMALL"):
        cases = [(64, 18, 20, 11)]
    rows = [run(*c) for c in cases]
    os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
    json.dump(rows, open(os.path.join(ROOT, "gpurun_out", "parity_report.json"), "w"), indent=1)
    for r in rows:
        print(f"## {r['B']} roots x {r['S']} simulations, A = {r['A']} (oracle: {r['tree_oracle']} ctree + PyTorch-CPU model, {r['oracle_seconds']} s)")
        for k, v in r.items():
            if k not in ("B", "A", "S", "tree_oracle", "oracle_seconds"):
                print(f"- {k}: {v}")


if __name__ == "__main__":
    main()
