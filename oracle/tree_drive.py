"""The reference search loops, written once, for every tree module the tests drive.  TEST INFRASTRUCTURE ONLY.

`drive(mod, case, kind, leaves)` runs one search of the reference driver protocol on `mod`: the compiled reference
(oracle/_ref), the C port (oracle.ctree_port / ctree_port_ez / ctree_port_stoch) or a device mirror (lightzero_b200.mz_tree /
ez_tree / gmz_tree / stochastic_mz_tree).  Kinds and the loops they restate:
  mz        MuZeroMCTSCtree.search                      mcts_ctree.py:267-368
  ez        EfficientZeroMCTSCtree.search               mcts_ctree.py:729-876    (is_reset = search_len % horizon == 0)
  reuse     MuZeroMCTSCtree.search_with_reuse           mcts_ctree.py:370-468    (compacted inference batch)
  ez_reuse  EfficientZeroMCTSCtree.search_with_reuse    mcts_ctree.py:878-1003
  gumbel    GumbelMuZeroMCTSCtree.search                mcts_ctree.py:1104-1172
  stoch     StochasticMuZeroMCTSCtree.search            mcts_ctree_stochastic.py:117-252  (chance leaves backed up first,
            then decision leaves, each call with its leaf_idx_list)

A case is a dict with the key names of the committed fixtures (tests/golden), so `np.load(fixture)` is a case:
B, A, S, legal (+ nlegal when padded), root_logits, to_play, and optionally use_noise / noise + noises, noise_w,
pb_c_base, pb_c_init, discount, delta, lstm_horizon_len, true_action / reuse_value (reuse kinds), m / root_values
(gumbel), C and chance_seed (stoch: None samples the chance draws from the tie hash key, which the port and the device
mirror support, the compiled reference does not), and the recorded leaf outputs rewards / values_in / policies (gumbel:
rewards / values / logits; stoch: policies max(A, C) wide).

`leaves(s, ix, iy, last_action, keep, mask)` gives simulation s's (reward or value prefix, value, policy logits) for
the batch rows `keep` (every row except the reuse kinds' no-inference ones); `mask` is the EfficientZero is_reset mask, or
for stoch the leaf_node_is_chance mask (the driver keeps the first C logits of a chance leaf's row, the first A of a
decision leaf's).  Three sources: `recorded(case, kind)`, `Sampled(draw)` and `network(model, latent, hidden)`.
"""
import numpy as np

PER_SIM = ("ix", "iy", "last_action", "search_len", "virtual_to_play", "is_reset", "n_inferred", "no_inference", "reuse_list",
           "is_chance")


def legal_lists(c):
    """A case's legal lists; a [B, A] uint8 / bool mask (the mirrors take one) passes through."""
    if isinstance(c["legal"], np.ndarray) and c["legal"].dtype in (np.uint8, np.bool_):
        return c["legal"]
    if "nlegal" in c:
        return [c["legal"][b, :c["nlegal"][b]].tolist() for b in range(int(c["B"]))]
    return [list(l) for l in c["legal"]]


def fixture_kind(d):
    if "C" in d:
        return "stoch"
    if "m" in d:
        return "gumbel"
    H = int(d["lstm_horizon_len"]) if "lstm_horizon_len" in d else 0
    return ("ez_reuse" if H else "reuse") if "true_action" in d else ("ez" if H else "mz")


def make_roots(mod, B, legal, A, S, horizon=5, C=None, chance_seed=None):
    """Roots of any tree module: the port takes its action space and node budget, ez_tree.Roots the LSTM horizon, the
    Stochastic MuZero modules the chance space (and the compiled reference the pinned random_device of chance_seed)."""
    name = mod.__name__
    if C is not None:
        if name == "oracle.ctree_port_stoch":
            roots = mod.Roots(B, legal, C, max_sims=S, action_space_size=A)
            if chance_seed is not None:
                from lightzero_b200.stochastic_mz_tree import chance_uniform
                roots.set_chance_u(chance_uniform(chance_seed))
            return roots
        if name == "lightzero_b200.stochastic_mz_tree":
            return mod.Roots(B, legal, C, chance_seed=chance_seed, max_simulations=S)
        if name != "stochastic_mz_tree":
            raise ValueError(f"{name} has no chance nodes: a Stochastic MuZero case runs on oracle.ctree_port_stoch, "
                             "lightzero_b200.stochastic_mz_tree or the compiled stochastic_mz_tree")
        if chance_seed is None:
            raise ValueError("the compiled reference tree draws its chance outcomes from a pinned random_device only")
        from oracle import build_stoch_ref
        build_stoch_ref.set_random_device(chance_seed)
        return mod.Roots(B, legal, C)
    if name.startswith("oracle.ctree_port"):
        return mod.Roots(B, legal, action_space_size=A, max_sims=S)
    if name == "lightzero_b200.ez_tree":
        return mod.Roots(B, legal, lstm_horizon_len=horizon)
    return mod.Roots(B, legal)


def _f32(x):
    return np.asarray(x, np.float32)


def recorded(c, kind="mz"):
    """The leaf outputs a case recorded.  Reuse kinds feed the compacted batch: the first n_inferred rows of a fixture,
    or the kept rows of a case that holds every row."""
    keys = ("rewards", "values", "logits") if kind == "gumbel" else ("rewards", "values_in", "policies")

    def leaves(s, ix, iy, la, keep, reset):
        out = [_f32(c[k][s]) for k in keys]
        if kind in ("reuse", "ez_reuse"):
            sel = slice(0, int(c["n_inferred"][s])) if "n_inferred" in c else keep
            out = [x[sel] for x in out]
        return [x.tolist() for x in out]
    return leaves


def random_case(B, A, S, seed, masks, noise, two_player, scale, reuse=False, horizon=0, C=None, chance_seed=None):
    """Seeded random inputs, drawn in this order: legal lists (60 % of the actions when masks, never empty), root
    logits, to_play, for ReZero the true actions and reuse values, then Dirichlet noise.  Returns the case and a Sampled
    source that goes on drawing r, v, p (normal, times scale) per simulation from the same generator.  C: a Stochastic
    MuZero case, whose policies are max(A, C) wide."""
    rng = np.random.default_rng(seed)
    legal = []
    for _ in range(B):
        m = rng.random(A) < 0.6 if masks else np.ones(A, bool)
        if not m.any():
            m[rng.integers(A)] = True
        legal.append(np.nonzero(m)[0].tolist())

    def normal(shape):
        return (rng.standard_normal(shape) * scale).astype(np.float32)
    c = dict(B=B, A=A, S=S, use_noise=noise, legal=legal, root_logits=normal((B, A)), lstm_horizon_len=horizon)
    c["to_play"] = rng.integers(1, 3, size=B).astype(np.int32) if two_player else np.full(B, -1, np.int32)
    if reuse:
        c["true_action"] = np.asarray([int(l[rng.integers(len(l))]) for l in legal], np.int32)
        c["reuse_value"] = normal(B)
    c["noises"] = np.zeros((B, A), np.float32)
    if noise:
        for b, l in enumerate(legal):
            c["noises"][b, :len(l)] = rng.dirichlet([0.3] * len(l)).astype(np.float32)
    if C is not None:
        c.update(C=C, chance_seed=chance_seed)
    W = A if C is None else max(A, C)
    return c, Sampled(lambda: (normal(B), normal(B), normal((B, W))))


class Sampled:
    """Leaf outputs drawn per simulation by draw() -> (r, v, p) over the whole batch; reuse kinds feed the first
    len(keep) rows.  `drawn` keeps every full draw (the fixtures store them padded to B rows)."""

    def __init__(self, draw):
        self.draw, self.drawn = draw, []

    def __call__(self, s, ix, iy, la, keep, reset):
        out = self.draw()
        self.drawn.append(out)
        return [x[:len(keep)].tolist() for x in out]


def network(model, latent, hidden=None, zero_reset_state=True, stochastic=False):
    """A CUDA model evaluating the gathered leaves with return_scalars=True.  Latents (and for EfficientZero the LSTM
    state (h, c), each [B, H]) are kept per simulation and gathered at (ix, iy); the state stored for a reset leaf is
    zeroed (mcts_ctree.py:856-863) unless zero_reset_state is False.  stochastic: a StochasticMuZeroModelMLP, whose chance
    leaves (odd depth) run recurrent_inference(afterstate=False) and the others afterstate=True
    (mcts_ctree_stochastic.py:171-212)."""
    import torch
    pool = [latent]
    hpool = [hidden] if hidden is not None else None

    @torch.no_grad()
    def stoch_leaves(s, ix, iy, la, keep, is_chance):
        ixs, iys = np.asarray(ix)[keep], torch.as_tensor(np.asarray(iy)[keep], device=latent.device)
        lat = torch.empty((len(keep),) + tuple(latent.shape[1:]), device=latent.device, dtype=latent.dtype)
        for x in np.unique(ixs):            # gather the leaves' parents slot by slot
            rows = torch.as_tensor(np.nonzero(ixs == x)[0], device=latent.device)
            lat[rows] = pool[int(x)][iys[rows]]
        act = torch.tensor([la[k] for k in keep], device=lat.device)
        nxt = torch.zeros_like(lat)
        r, v, p = [0.0] * len(keep), [0.0] * len(keep), [None] * len(keep)
        for chance in (True, False):
            sel = [k for k in keep if bool(is_chance[k]) == chance]
            if not sel:
                continue
            o = model.recurrent_inference(lat[sel], act[sel], afterstate=not chance, return_scalars=True)
            nxt[sel] = o.latent_state
            for k, rk, vk, pk in zip(sel, o.reward_scalar.cpu().tolist(), o.value_scalar.cpu().tolist(),
                                     o.policy_logits.cpu().tolist()):
                r[k], v[k], p[k] = rk, vk, pk
        pool.append(nxt)
        return r, v, p

    @torch.no_grad()
    def leaves(s, ix, iy, la, keep, reset):
        if stochastic:
            return stoch_leaves(s, ix, iy, la, keep, reset)
        if not keep:
            pool.append(None)
            if hpool is not None:
                hpool.append(None)
            return [], [], []
        lat = torch.stack([pool[ix[k]][iy[k]] for k in keep])
        act = torch.tensor([la[k] for k in keep], device=lat.device)
        if hpool is None:
            o = model.recurrent_inference(lat, act, return_scalars=True)
            r = o.reward_scalar
        else:
            h, c = (torch.stack([hpool[ix[k]][i][iy[k]] for k in keep]) for i in (0, 1))
            o = model.recurrent_inference(lat, (h[None], c[None]), act, return_scalars=True)
            r = o.value_prefix_scalar
            zero = torch.from_numpy(reset[keep] & zero_reset_state).to(lat.device).view(-1, 1)
            hpool.append(tuple(torch.where(zero, 0.0, o.reward_hidden_state[i][0]) for i in (0, 1)))
        pool.append(o.latent_state)
        return r.cpu().tolist(), o.value_scalar.cpu().tolist(), o.policy_logits.cpu().tolist()
    return leaves


def from_recorder(rec):
    """oracle/search_ref.py's per-simulation records under the case and trace key names"""
    keys = dict(reward="rewards", value="values_in", policy="policies")
    return {keys.get(k, k): [r[k] for r in rec] for k in rec[0]}


def _pad(rows, width):
    out = np.full((len(rows), width), -1, np.int32)
    for b, r in enumerate(rows):
        out[b, :len(r)] = r
    return out


def readout(roots, A, S, gumbel_discount=None):
    """The final read-outs of any Roots: visit counts and trajectories -1 padded, root values as fp32 bits, and for
    Gumbel roots the improved policies and completed children values."""
    out = dict(distributions=_pad(roots.get_distributions(), A),
               root_values_bits=_f32(roots.get_values()).view(np.uint32),
               trajectories=_pad(roots.get_trajectories(), S + 1))
    if gumbel_discount is not None:
        out["policies"] = _f32(roots.get_policies(gumbel_discount, A))
        out["children_values"] = _f32(roots.get_children_values(gumbel_discount, A))
    return out


def drive(mod, c, kind, leaves, det=True, setup=None, reset_in_backup=True):
    """One search of `kind` on tree module `mod` with the inputs of case `c` and leaf outputs from `leaves`.
    det: the MuZero descents' deterministic flag.  setup(roots) runs after prepare (tie-hash mode, device tie-break).
    reset_in_backup=False withholds is_reset from the EfficientZero back-up (a sensitivity mutant).
    Returns (trace, roots): the trace holds per simulation ix, iy, last_action, search_len, virtual_to_play, and
    is_reset (ez kinds) or n_inferred, no_inference, reuse_list (reuse kinds), each [S, B] ([S] / [S, B + 1]); then
    the readout()."""
    B, A, S = int(c["B"]), int(c["A"]), int(c["S"])
    gumbel, ez, reuse, stoch = kind == "gumbel", kind in ("ez", "ez_reuse"), kind in ("reuse", "ez_reuse"), kind == "stoch"
    C = int(c["C"]) if stoch else None
    chance_seed = c.get("chance_seed") if stoch else None
    if chance_seed is not None and np.ndim(chance_seed) == 0 and int(chance_seed) < 0:
        chance_seed = None          # fixtures store a sampled case's chance_seed as -1
    chance_seed = None if chance_seed is None else int(chance_seed)
    disc = float(c.get("discount", 0.997))
    horizon = int(c.get("lstm_horizon_len", 5))
    legal = legal_lists(c)
    tp = c["to_play"]
    tp = [int(tp)] * B if np.ndim(tp) == 0 else [int(x) for x in tp]
    noises = None
    # noise switch: use_noise (tree / reuse fixtures), noise (Gumbel fixtures), else whether the case holds noises at all
    if int(c.get("use_noise", c.get("noise", "noises" in c and c["noises"] is not None))):
        noises = [_f32(c["noises"][b][:len(l)]).tolist() for b, l in enumerate(legal)]
    logits = _f32(c["root_logits"]).tolist()
    pre = [_f32(c["root_values"]).tolist()] if gumbel else []
    roots = make_roots(mod, B, legal, A, S, horizon, C, chance_seed)
    if noises is None:
        roots.prepare_no_noise([0.] * B, *pre, logits, tp)
    else:
        roots.prepare(float(c.get("noise_w", 0.25)), noises, [0.] * B, *pre, logits, tp)
    if mod.__name__ in ("lightzero_b200.mz_tree", "lightzero_b200.ez_tree"):
        roots._materialize(S)          # node pool sized to this search (gmz_tree sizes its trees at the first descent)
    if setup is not None:
        setup(roots)
    mm = mod.MinMaxStatsList(B)
    mm.set_delta(float(c.get("delta", 0.01)))
    pbc = (int(c.get("pb_c_base", 19652)), float(c.get("pb_c_init", 1.25)), disc, mm)
    if reuse:
        ta, rv = [int(x) for x in c["true_action"]], _f32(c["reuse_value"]).tolist()
    t = {k: [] for k in PER_SIM}
    for s in range(S):
        res = mod.ResultsWrapper(B)
        if gumbel:
            ix, iy, la, vtp = mod.batch_traverse(roots, S, int(c["m"]), disc, res, list(tp))
        elif reuse:
            ix, iy, la, vtp = mod.batch_traverse_with_reuse(roots, *pbc, res, list(tp), ta, rv)
        elif ez:
            ix, iy, la, vtp = mod.batch_traverse(roots, *pbc, res, list(tp))
        elif stoch:        # the compiled reference has no deterministic switch (rand() == 0: the first maximum)
            kw = {} if mod.__name__ == "stochastic_mz_tree" else dict(deterministic=det)
            ch, ix, iy, la, vtp = mod.batch_traverse(roots, *pbc, res, list(tp), **kw)
            ch = np.asarray([bool(x) for x in ch])
            t["is_chance"].append(ch.astype(np.int32))
        else:
            ix, iy, la, vtp = mod.batch_traverse(roots, *pbc, res, list(tp), det)
        ix, iy, la, vtp = list(ix), list(iy), list(la), list(vtp)
        slen = list(res.get_search_len())
        for k, v in zip(PER_SIM, (ix, iy, la, slen, vtp)):
            t[k].append(v)
        reset = (np.asarray(slen) % horizon == 0) if ez else (ch if stoch else None)
        keep = [k for k in range(B) if ix[k] != -1]
        r, v, p = leaves(s, ix, iy, la, keep, reset)
        args = (s + 1, disc, r, v, p, mm, res)
        rs = []
        if ez:
            t["is_reset"].append(reset.astype(np.int32))
            rs = [(reset if reset_in_backup else np.zeros(B, bool)).astype(np.int32).tolist()]
        if gumbel:
            mod.batch_back_propagate(*args, vtp)
        elif stoch:        # chance leaves first, then decision leaves (mcts_ctree_stochastic.py:229-252)
            for chance in (True, False):
                idx = [k for k in range(B) if ch[k] == chance]
                if idx:
                    rows = [list(p[k])[:C if chance else A] for k in idx]
                    mod.batch_backpropagate(s + 1, disc, [r[k] for k in idx], [v[k] for k in idx], rows, mm, res, vtp,
                                            [bool(x) for x in ch], idx)
        elif reuse:        # no_inference_lst / reuse_lst as the driver builds them, -1 terminated
            no_inf = [iy[k] for k in range(B) if ix[k] == -1]
            reuse_lst = [k for k in range(B) if ix[k] == 0 and la[k] == ta[k]]
            t["n_inferred"].append(len(keep))
            t["no_inference"].append(no_inf)
            t["reuse_list"].append(reuse_lst)
            mod.batch_backpropagate_with_reuse(*args, *rs, vtp, no_inf + [-1], reuse_lst + [-1], rv)
        else:
            mod.batch_backpropagate(*args, *rs, vtp)
    trace = {k: np.asarray(v, np.int32) for k, v in t.items() if v and k not in ("no_inference", "reuse_list")}
    if reuse:
        trace["no_inference"], trace["reuse_list"] = _pad(t["no_inference"], B + 1), _pad(t["reuse_list"], B + 1)
    trace.update(readout(roots, A, S, disc if gumbel else None))
    return trace, roots


def fixture_trace(d):
    """What a committed fixture expects, under the trace's key names (the Gumbel fixtures store exp_* arrays)."""
    if "exp_rec" in d:
        t = dict(zip(PER_SIM[:5], d["exp_rec"]))
        t.update(distributions=d["exp_dist"], root_values_bits=d["exp_root_value"].view(np.uint32),
                 trajectories=d["exp_traj"], policies=d["exp_policy"], children_values=d["exp_children_values"])
        return t
    t = {k: d[k] for k in PER_SIM + ("distributions", "root_values_bits", "trajectories") if k in d}
    if fixture_kind(d) == "reuse":      # the MuZero reuse fixtures store an all-zero is_reset the loop never computes
        del t["is_reset"]
    return t


def check_fixture(mod, d):
    """Replays fixture d through tree module `mod` with the leaf outputs it recorded and asserts that every per-simulation
    and final array the fixture holds comes out identical.  Returns (trace, roots)."""
    kind = fixture_kind(d)
    trace, roots = drive(mod, d, kind, recorded(d, kind))
    exp = fixture_trace(d)
    assert {"distributions", "root_values_bits", "search_len"} <= set(exp) <= set(trace), (sorted(exp), sorted(trace))
    assert_same(trace, exp)
    return trace, roots


def _bits(x):
    x = np.asarray(x)
    return x.view(np.uint32) if x.dtype == np.float32 else x


def assert_same(got, exp):
    """Every array the two traces (or a trace and fixture_trace) share is identical; floats compare as bits.  A
    per-simulation mismatch names the first simulation that differs."""
    for k in got:
        if k not in exp:
            continue
        g, e = _bits(got[k]), _bits(exp[k])
        if k in PER_SIM and g.shape == e.shape and g.ndim > 0 and not np.array_equal(g, e):
            s = int(np.nonzero([not np.array_equal(a, b) for a, b in zip(g, e)])[0][0])
            raise AssertionError(f"{k} differs first at simulation {s}: {g[s].tolist()} != {e[s].tolist()}")
        assert np.array_equal(g, e), k
