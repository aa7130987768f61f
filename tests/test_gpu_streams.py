"""Every entry point on the caller's own stream, next to a busy legacy default stream (INTEGRATION.md, Streams).

The training-loop layout this covers: a learner keeps the legacy default stream busy while a collector runs the library on a
torch.cuda.Stream() of its own.  Such streams are non-blocking: nothing orders them against the default stream, so a library
write left on the default stream lands after the kernels that read it, and a library call that waits for the default stream
stalls the collector behind the learner.

Harness (_check_on_side_stream), per scenario:
  1. run it on the default stream and keep its outputs (also the timed dry run);
  2. queue torch.cuda._sleep on the default stream, about 3x the dry run (at most ~5 s), and record an event after it;
  3. run the same scenario, object creation to read-back, inside torch.cuda.stream(side), device outputs copied to pinned host
     memory on `side`;
  4. synchronise `side` only;
  5. the default-stream event has not completed (no call waited for the default stream), and the outputs equal step 1 bit for
     bit;
  6. synchronise the device.
Scenarios that grow a live workspace or reload weights free device memory, and cudaFree waits for the whole device (documented
in INTEGRATION.md): they check the values only.  For the same reason every scenario hands the objects it created back under
"_keep", and they are destroyed after the checks."""
import gc
import time

import numpy as np
import pytest
import torch

import board_model_ref as BR
import mlp_ez_model_ref as ER
import mlp_fp32_model_ref as FR
import mlp_mz_model_ref as MR
from test_gpu_search_oracle import _inputs

pytestmark = pytest.mark.gpu

DISCOUNT = 0.997


@pytest.fixture(scope="module")
def sleep_rate():
    """torch.cuda._sleep cycles per second on this device (a bounded spin kernel)"""
    torch.cuda._sleep(1_000_000)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    torch.cuda._sleep(100_000_000)
    b.record()
    b.synchronize()
    return 100_000_000 / (a.elapsed_time(b) * 1e-3)


def _host(v):
    """numpy copy of a scenario output (device tensors, host tensors, lists, scalars)"""
    if isinstance(v, torch.Tensor):
        return v.detach().cpu().numpy()
    return np.asarray(v)


def _same_bits(got, ref, name):
    assert got.keys() == ref.keys(), name
    for k in ref:
        a, b = np.ascontiguousarray(got[k]), np.ascontiguousarray(ref[k])
        assert a.dtype == b.dtype and a.shape == b.shape, (name, k, a.dtype, b.dtype, a.shape, b.shape)
        same = a.view(np.uint8).reshape(a.shape + (-1,)) == b.view(np.uint8).reshape(b.shape + (-1,)) if a.size else np.ones(0, bool)
        assert same.all(), "%s: output %r differs from the default-stream run at %d of %d elements" % (
            name, k, int((~same.reshape(a.size, -1).all(1)).sum()), a.size)


def _check_on_side_stream(rate, name, scenario, syncs_device=False):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = scenario()
    out.pop("_keep", None)
    ref = {k: _host(v) for k, v in out.items()}
    torch.cuda.synchronize()
    dry = time.perf_counter() - t0
    assert dry < 1.6, "%s: the dry run took %.2f s, longer than the busy window covers" % (name, dry)
    # pinned read-back buffers allocated before the window
    pinned = {k: torch.empty(v.shape, dtype=v.dtype, pin_memory=True) for k, v in out.items() if isinstance(v, torch.Tensor) and v.is_cuda}
    del out
    side = torch.cuda.Stream()
    gc.collect()          # no garbage collection (and so no destroy of an earlier run's objects) inside the window
    gc.disable()
    torch.cuda.synchronize()
    torch.cuda._sleep(int(min(max(3.0 * dry, 0.3), 5.0) * rate))     # the learner's backward pass
    busy = torch.cuda.Event()
    busy.record()
    with torch.cuda.stream(side):
        out = scenario()
        keep = out.pop("_keep", None)      # destroyed after the checks: a destroy frees memory, and cudaFree waits for the device
        got = {}
        for k, v in out.items():
            if k in pinned:
                got[k] = pinned[k].copy_(v, non_blocking=True)
            else:
                got[k] = v
    side.synchronize()
    still_busy = not busy.query()
    torch.cuda.synchronize()
    gc.enable()
    del keep
    if not syncs_device:
        assert still_busy, "%s: a library call waited for the legacy default stream" % name
    _same_bits({k: _host(v) for k, v in got.items()}, ref, name)
    return ref


# ---- inputs, built once on the host ----
def _conv_sd(obs, A, seed, ez=False):
    from oracle import model_ref as R
    ref = R.EfficientZeroModelRef(obs, A) if ez else R.MuZeroModelRef(obs, A)
    return {k: v.clone() for k, v in R.emulate_trained_(ref, seed).state_dict().items()}


def _search_inputs(B, A, seed, players="1p"):
    legal, _, noises, tp = _inputs(B, A, seed, players)
    return legal, noises, tp


def _readout(roots, A, S, gumbel=False):
    from oracle.tree_drive import readout
    return readout(roots, A, S, DISCOUNT if gumbel else None)


# ---- the conv model's entry points: initial inference (workspace zeroed on the caller's stream), recurrent, the transform.
# The workspace's pads come out of cudaMalloc zero on an H100 even after other buffers were freed there, so a workspace memset
# left on the legacy stream would still give the right values here: tests/test_streams_cpu.py is what guards that call ----
@pytest.mark.parametrize("B", [1, 8])
def test_conv96_inference_on_side_stream(sleep_rate, B):
    import lightzero_b200 as lzb
    A, obs_shape = 18, (4, 96, 96)
    sd = _conv_sd(obs_shape, A, 3)
    x = torch.rand((B,) + obs_shape, generator=torch.Generator().manual_seed(1)).cuda()
    act = torch.arange(B, dtype=torch.int64).remainder(A).cuda()

    def scenario():
        m = lzb.MuZeroModel(observation_shape=obs_shape, action_space_size=A).load_state_dict(sd)
        o = m.initial_inference(x)
        r = m.recurrent_inference(o.latent_state, act)
        inv = lzb.InverseScalarTransform(lzb.DiscreteSupport(-300., 301., 1.))
        return dict(latent=o.latent_state, logits=o.policy_logits, value=o.value, next_latent=r.latent_state,
                    reward=r.reward, rvalue=r.value, rlogits=r.policy_logits, scalar=inv(o.value), _keep=(m, inv))

    _check_on_side_stream(sleep_rate, "conv96 B=%d" % B, scenario)


def test_conv96_workspace_growth_on_side_stream(sleep_rate):
    """B = 8 and then B = 1024: the growth frees the B = 8 workspace (a device-wide wait) and zeroes the new one on `side`"""
    import lightzero_b200 as lzb
    A, obs_shape = 18, (4, 96, 96)
    sd = _conv_sd(obs_shape, A, 5)
    x = torch.rand((1024,) + obs_shape, generator=torch.Generator().manual_seed(2)).cuda()

    def scenario():
        m = lzb.MuZeroModel(observation_shape=obs_shape, action_space_size=A).load_state_dict(sd)
        small = m.initial_inference(x[:8])
        big = m.initial_inference(x)
        return dict(small=small.latent_state, small_logits=small.policy_logits, big=big.latent_state,
                    big_logits=big.policy_logits, big_value=big.value, _keep=m)

    _check_on_side_stream(sleep_rate, "conv96 growth", scenario, syncs_device=True)


# ---- the fused searches: model, tree and search created on `side`.  Deterministic ties: stochastic ones draw from the pooled
# tree's RNG epoch, which every reset advances, so a second search on the same inputs would break ties differently ----
def _mz_search(make_model, x, A, S, seed, players="1p", reuse=False):
    import lightzero_b200 as lzb
    B = x.shape[0]
    legal, noises, tp = _search_inputs(B, A, seed, players)
    rng = np.random.default_rng(seed)
    true_action = [int(l[rng.integers(len(l))]) for l in legal]
    reuse_value = (rng.standard_normal(B) * 0.5).astype(np.float32).tolist()

    def scenario():
        m = make_model()
        o = m.initial_inference(x)
        mcts = lzb.MuZeroMCTSCtree(dict(num_simulations=S, deterministic=True, discount_factor=DISCOUNT))
        roots = mcts.roots(B, legal)
        roots.prepare(0.25, noises, [0.] * B, o.policy_logits, tp)
        if reuse:
            mcts.search_with_reuse(roots, m, o.latent_state, tp, true_action, reuse_value)
        else:
            mcts.search(roots, m, o.latent_state, tp)
        out = _readout(roots, A, S)
        roots.clear()
        out["_keep"] = (m, mcts)
        return out
    return scenario


def _conv_model(obs_shape, A, seed):
    import lightzero_b200 as lzb
    sd = _conv_sd(obs_shape, A, seed)
    return lambda: lzb.MuZeroModel(observation_shape=obs_shape, action_space_size=A, downsample=True).load_state_dict(sd)


def _rand(shape, seed):
    return torch.rand(shape, generator=torch.Generator().manual_seed(seed)).cuda()


@pytest.mark.parametrize("case", ["persistent_a6", "graph_a33", "reuse_a6"])
def test_muzero_search_on_side_stream(sleep_rate, case):
    A = 33 if case == "graph_a33" else 6
    x = _rand((24, 4, 84, 84), 7)
    _check_on_side_stream(sleep_rate, case, _mz_search(_conv_model((4, 84, 84), A, 11), x, A, 10, 13, reuse=case.startswith("reuse")))


def test_board_search_on_side_stream(sleep_rate):
    import lightzero_b200 as lzb
    sd = BR.build("tictactoe", 2).state_dict()
    x = _rand((16,) + tuple(BR.BOARD_CONFIGS["tictactoe"][0]), 8)
    make = lambda: lzb.MuZeroModel(**BR.model_kwargs("tictactoe")).load_state_dict(sd)
    _check_on_side_stream(sleep_rate, "tictactoe", _mz_search(make, x, 9, 10, 14, players="2p"))


@pytest.mark.parametrize("name, kernel", [("cartpole", "fp32"), ("lunarlander", "tc")])
def test_mlp_search_on_side_stream(sleep_rate, name, kernel):
    import lightzero_b200 as lzb
    ref_mod = FR if kernel == "fp32" else MR
    sd = ref_mod.build(name, 3).state_dict()
    kw = ref_mod.model_kwargs(name)
    x = _rand((16, ref_mod.CONFIGS[name][0]), 9)
    make = lambda: lzb.MuZeroModelMLP(**kw).load_state_dict(sd)
    _check_on_side_stream(sleep_rate, "mlp " + name, _mz_search(make, x, ref_mod.CONFIGS[name][1], 10, 15))


def _ez_search(make_model, x, A, S, seed):
    import lightzero_b200 as lzb
    B = x.shape[0]
    legal, noises, _ = _search_inputs(B, A, seed)

    def scenario():
        m = make_model()
        o = m.initial_inference(x)
        mcts = lzb.EfficientZeroMCTSCtree(dict(num_simulations=S, lstm_horizon_len=3, discount_factor=DISCOUNT))
        roots = mcts.roots(B, legal)
        roots.prepare(0.25, noises, [0.] * B, o.policy_logits, [-1] * B)
        mcts.search(roots, m, o.latent_state, o.reward_hidden_state, [-1] * B)
        out = _readout(roots, A, S)
        roots.clear()
        out["_keep"] = (m, mcts)
        return out
    return scenario


def test_efficientzero_conv_search_on_side_stream(sleep_rate):
    import lightzero_b200 as lzb
    sd = _conv_sd((4, 96, 96), 6, 6, ez=True)
    make = lambda: lzb.EfficientZeroModel(observation_shape=(4, 96, 96), action_space_size=6).load_state_dict(sd)
    _check_on_side_stream(sleep_rate, "ez conv", _ez_search(make, _rand((16, 4, 96, 96), 10), 6, 10, 16))


def test_efficientzero_mlp_search_on_side_stream(sleep_rate):
    import lightzero_b200 as lzb
    sd = ER.build("cartpole", 4).state_dict()
    make = lambda: lzb.EfficientZeroModelMLP(**ER.model_kwargs("cartpole")).load_state_dict(sd)
    _check_on_side_stream(sleep_rate, "ez mlp", _ez_search(make, _rand((16, 4), 11), 2, 10, 17))


def test_gumbel_search_on_side_stream(sleep_rate):
    import lightzero_b200 as lzb
    B, A, S = 16, 6, 10
    make = _conv_model((4, 64, 64), A, 12)
    x = _rand((B, 4, 64, 64), 12)
    legal, noises, tp = _search_inputs(B, A, 18)

    def scenario():
        m = make()
        o = m.initial_inference(x, return_scalar_value=True)
        mcts = lzb.GumbelMuZeroMCTSCtree(dict(num_simulations=S, max_num_considered_actions=4, discount_factor=DISCOUNT))
        roots = mcts.roots(B, legal)
        roots.prepare(0.25, noises, [0.0] * B, o.value_scalar, o.policy_logits, tp)
        mcts.search(roots, m, o.latent_state, tp)
        out = _readout(roots, A, S, gumbel=True)
        roots.clear()
        out["_keep"] = (m, mcts)
        return out
    _check_on_side_stream(sleep_rate, "gumbel", scenario)


# ---- collect: device and host-chunked paths, device select_action, a pooled tree switched MuZero -> Gumbel -> MuZero ----
def _collect_inputs(B, A, seed):
    rng = np.random.default_rng(seed)
    mask = (rng.random((B, A)) < 0.7).astype(np.uint8)
    mask[np.arange(B), rng.integers(0, A, B)] = 1
    noise = rng.dirichlet([0.3] * A, size=B).astype(np.float32)
    return mask, noise


@pytest.mark.parametrize("kind", ["muzero", "gumbel"])
@pytest.mark.parametrize("path", ["device", "host"])
def test_collect_on_side_stream(sleep_rate, kind, path):
    import lightzero_b200 as lzb
    B, A, S = 24, 6, 8
    make = _conv_model((4, 64, 64), A, 13)
    x = torch.rand((B, 4, 64, 64), generator=torch.Generator().manual_seed(13))
    mask, noise = _collect_inputs(B, A, 19)
    if path == "device":
        x, mask, noise = x.cuda(), torch.from_numpy(mask).cuda(), torch.from_numpy(noise).cuda()
    else:
        x, mask, noise = x.pin_memory(), torch.from_numpy(mask), torch.from_numpy(noise)
    cfg = dict(num_simulations=S, discount_factor=DISCOUNT)

    def scenario():
        m = make()
        if kind == "gumbel":
            pol = lzb.GumbelMuZeroCollectPolicy(m, dict(cfg, max_num_considered_actions=4))
        else:
            pol = lzb.MuZeroCollectPolicy(m, dict(cfg, deterministic=True))
        r = pol.search_batch(x, mask, noise, read_back=False, select=(1.0, False, 5))
        return dict({k: v.clone() for k, v in r.items()}, _keep=(m, pol))
    _check_on_side_stream(sleep_rate, "collect %s %s" % (kind, path), scenario)


def test_pooled_tree_switch_on_side_stream(sleep_rate):
    """one pooled tree serves MuZero, Gumbel, MuZero and Gumbel collects: switching it back to MuZero keeps the Gumbel state
    idle (no free), and the second Gumbel collect re-attaches it.  B = 20 is a pool key no other test uses, so the first Gumbel
    collect of the default-stream run attaches fresh state: the re-attached one must give the same bits"""
    import lightzero_b200 as lzb
    B, A, S = 20, 6, 8
    make = _conv_model((4, 64, 64), A, 14)
    x = _rand((B, 4, 64, 64), 14)
    mask, noise = _collect_inputs(B, A, 20)
    mask, noise = torch.from_numpy(mask).cuda(), torch.from_numpy(noise).cuda()
    cfg = dict(num_simulations=S, discount_factor=DISCOUNT)

    def scenario():
        m = make()
        mz = lzb.MuZeroCollectPolicy(m, dict(cfg, deterministic=True))
        gz = lzb.GumbelMuZeroCollectPolicy(m, dict(cfg, max_num_considered_actions=4))
        out = {}
        for tag, pol in (("mz0", mz), ("gz", gz), ("mz1", mz), ("gz1", gz)):
            r = pol.search_batch(x, mask, noise, read_back=False, select=(1.0, True, 0))
            out.update({tag + "_" + k: v.clone() for k, v in r.items()})
        out["_keep"] = (m, mz, gz)
        return out
    ref = _check_on_side_stream(sleep_rate, "pooled tree switch", scenario)
    _same_bits({k[4:]: v for k, v in ref.items() if k.startswith("gz1_")}, {k[3:]: v for k, v in ref.items() if k.startswith("gz_")},
               "re-attached Gumbel state vs fresh")
    _same_bits({k[4:]: v for k, v in ref.items() if k.startswith("mz1_")}, {k[4:]: v for k, v in ref.items() if k.startswith("mz0_")},
               "MuZero collect after a Gumbel one")


# ---- reanalyze and the collector's device state ----
def test_reanalyze_on_side_stream(sleep_rate):
    import lightzero_b200 as lzb
    from lightzero_b200.reanalyze import compute_target_policy_reanalyzed
    T, A, S, K = 24, 6, 8, 5
    make = _conv_model((4, 84, 84), A, 15)
    x = _rand((T, 4, 84, 84), 15)
    _, noise = _collect_inputs(T, A, 21)
    mask = np.ones((T, A), np.uint8)                  # fixed_action_space: every action legal
    to_play, policy_mask = [-1] * T, [1] * (T - 2) + [0, 0]

    def scenario():
        m = make()
        mcts = lzb.MuZeroMCTSCtree(dict(num_simulations=S, deterministic=True, discount_factor=DISCOUNT))
        t = compute_target_policy_reanalyzed(m, mcts, x, mask, to_play, policy_mask, [0, 0, 0, 0], num_unroll_steps=K,
                                             action_space_size=A, noises=noise)
        return dict(target=np.asarray(t, np.float32), _keep=(m, mcts))
    _check_on_side_stream(sleep_rate, "reanalyze", scenario)


def test_collector_state_on_side_stream(sleep_rate):
    """FrameStack and SegmentStats created on `side` (their zeroing: the setup stream), fed by a Gumbel collect whose improved
    policies go into the segments' improved-policy array"""
    import lightzero_b200 as lzb
    from lightzero_b200.collector import FrameStack, SegmentStats
    B, A, S, T = 16, 6, 8, 4
    make = _conv_model((4, 64, 64), A, 16)
    rng = np.random.default_rng(22)
    frames = [torch.from_numpy(rng.integers(0, 256, (B, 64, 64), dtype=np.uint8)).pin_memory() for _ in range(3)]
    resets = [torch.from_numpy(r).pin_memory() for r in (np.ones(B, np.uint8), (rng.random(B) < 0.3).astype(np.uint8),
                                                          np.zeros(B, np.uint8))]
    mask, noise = _collect_inputs(B, A, 23)
    mask, noise = torch.from_numpy(mask).cuda(), torch.from_numpy(noise).cuda()
    done = torch.from_numpy((rng.random(B) < 0.4).astype(np.uint8)).cuda()

    def scenario():
        m = make()
        pol = lzb.GumbelMuZeroCollectPolicy(m, dict(num_simulations=S, max_num_considered_actions=4, discount_factor=DISCOUNT))
        fs, seg = FrameStack(B, 4, 64, 64), SegmentStats(B, T, A)
        out = {}
        for i, (f, r) in enumerate(zip(frames, resets)):
            fs.push(f, reset=r)
            res = pol.search_batch(fs.view(), mask, noise, read_back=False, select=(1.0, True, i))
            seg.store_search_stats(res["visits"], res["values"], improved_policy=res["improved_policy"])
            if i == 1:
                seg.reset(done)
            out["obs%d" % i] = fs.view().clone()
        cv, rv, ln = seg.tensors()
        out.update(child_visits=cv.clone(), root_values=rv.clone(), lengths=ln.clone(), improved=seg.improved_policy().clone())
        out["_keep"] = (m, pol, fs, seg)
        return out
    _check_on_side_stream(sleep_rate, "collector", scenario)


# ---- concurrency: two independent sets on two streams, and one model shared by two searches ordered with events ----
def test_two_independent_searches_interleaved_on_two_streams(sleep_rate):
    import lightzero_b200 as lzb
    B, S = 16, 8
    sets = []
    for i, A in enumerate((6, 18)):
        sd = _conv_sd((4, 84, 84), A, 30 + i)
        legal, noises, _ = _search_inputs(B, A, 40 + i)
        sets.append((A, sd, _rand((B, 4, 84, 84), 50 + i), legal, noises))

    def run(streams):
        st = [dict() for _ in sets]
        steps = [
            lambda c, s: c.update(m=lzb.MuZeroModel(observation_shape=(4, 84, 84), action_space_size=s[0]).load_state_dict(s[1])),
            lambda c, s: c.update(o=c["m"].initial_inference(s[2])),
            lambda c, s: c.update(mcts=lzb.MuZeroMCTSCtree(dict(num_simulations=S, deterministic=True, discount_factor=DISCOUNT))),
            lambda c, s: c.update(roots=c["mcts"].roots(B, s[3])),
            lambda c, s: c["roots"].prepare(0.25, s[4], [0.] * B, c["o"].policy_logits, [-1] * B),
            lambda c, s: c["mcts"].search(c["roots"], c["m"], c["o"].latent_state, [-1] * B),
        ]
        for step in steps:                                # launches interleaved, no synchronisation between the sets
            for c, s, stream in zip(st, sets, streams):
                with torch.cuda.stream(stream):
                    step(c, s)
        out = {}
        for i, (c, s, stream) in enumerate(zip(st, sets, streams)):
            with torch.cuda.stream(stream):
                out.update({"%d_%s" % (i, k): v for k, v in _readout(c["roots"], s[0], S).items()})
                c["roots"].clear()
        out["_keep"] = st
        return out

    torch.cuda.synchronize()
    d = torch.cuda.current_stream()
    ref = run([d, d])
    ref.pop("_keep")
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    gc.collect()
    gc.disable()
    torch.cuda._sleep(int(3.0 * sleep_rate))
    busy = torch.cuda.Event()
    busy.record()
    got = run(streams)
    keep = got.pop("_keep")
    for s in streams:
        s.synchronize()
    still_busy = not busy.query()
    torch.cuda.synchronize()
    gc.enable()
    del keep
    assert still_busy, "a library call waited for the legacy default stream"
    _same_bits({k: _host(v) for k, v in got.items()}, {k: _host(v) for k, v in ref.items()}, "two streams")


def test_one_model_shared_by_two_searches_ordered_with_events(sleep_rate):
    """one lz_model's scratch serves two searches on two streams: the caller orders them with an event"""
    import lightzero_b200 as lzb
    B, A, S = 16, 6, 8
    sd = _conv_sd((4, 84, 84), A, 33)
    xs = [_rand((B, 4, 84, 84), 60 + i) for i in range(2)]
    inp = [_search_inputs(B, A, 70 + i) for i in range(2)]

    def run(s1, s2):
        with torch.cuda.stream(s1):
            m = lzb.MuZeroModel(observation_shape=(4, 84, 84), action_space_size=A).load_state_dict(sd)
        out, roots = {}, []
        prev = None
        for i, stream in enumerate((s1, s2)):
            with torch.cuda.stream(stream):
                if prev is not None:
                    stream.wait_event(prev)
                legal, noises, tp = inp[i]
                o = m.initial_inference(xs[i])
                mcts = lzb.MuZeroMCTSCtree(dict(num_simulations=S, deterministic=True, discount_factor=DISCOUNT))
                r = mcts.roots(B, legal)
                r.prepare(0.25, noises, [0.] * B, o.policy_logits, tp)
                mcts.search(r, m, o.latent_state, tp)
                roots.append((r, stream))
                prev = torch.cuda.Event()
                prev.record(stream)
        for i, (r, stream) in enumerate(roots):
            with torch.cuda.stream(stream):
                out.update({"%d_%s" % (i, k): v for k, v in _readout(r, A, S).items()})
                r.clear()
        out["_keep"] = m
        return out

    torch.cuda.synchronize()
    d = torch.cuda.current_stream()
    ref = run(d, d)
    ref.pop("_keep")
    torch.cuda.synchronize()
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    gc.collect()
    gc.disable()
    torch.cuda._sleep(int(3.0 * sleep_rate))
    busy = torch.cuda.Event()
    busy.record()
    got = run(s1, s2)
    keep = got.pop("_keep")
    s1.synchronize()
    s2.synchronize()
    still_busy = not busy.query()
    torch.cuda.synchronize()
    gc.enable()
    del keep
    assert still_busy, "a library call waited for the legacy default stream"
    _same_bits({k: _host(v) for k, v in got.items()}, {k: _host(v) for k, v in ref.items()}, "shared model")


# ---- pooled trees handed from one holder to the next while the first holder's search is still queued ----
def _collect_set(A, seed, B, **cfg):
    import lightzero_b200 as lzb
    m = _conv_model((4, 84, 84), A, seed)()
    pol = lzb.MuZeroCollectPolicy(m, dict(dict(num_simulations=30, deterministic=True, discount_factor=DISCOUNT), **cfg))
    mask, noise = _collect_inputs(B, A, seed)
    return m, pol, _rand((B, 4, 84, 84), seed), torch.from_numpy(mask).cuda(), torch.from_numpy(noise).cuda()


def _collect_once(s):
    _, pol, x, mask, noise = s
    r = pol.search_batch(x, mask, noise, read_back=False, select=(1.0, True, 0))
    return {k: v.clone() for k, v in r.items()}


def test_two_collects_of_one_shape_interleaved_on_two_streams(sleep_rate):
    """Two MuZeroCollectPolicy of the same (B, A, S), two models, on two side streams: search_batch(read_back=False) hands the
    pooled tree back while its search is still queued, and the other stream picks the same tree up.  Both streams are held by
    equal spin kernels, so without ordering the two searches would run at once on one tree."""
    B, A = 256, 18
    sets = [_collect_set(A, 80 + i, B) for i in range(2)]
    ref = [_collect_once(s) for s in sets]
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    for st in streams:
        with torch.cuda.stream(st):
            torch.cuda._sleep(int(0.1 * sleep_rate))
    got = []
    for s, st in zip(sets, streams):
        with torch.cuda.stream(st):
            got.append(_collect_once(s))
    torch.cuda.synchronize()
    for i in range(2):
        _same_bits({k: _host(v) for k, v in got[i].items()}, {k: _host(v) for k, v in ref[i].items()}, "set %d" % i)


def test_pooled_tree_parameter_change_waits_for_the_running_search(sleep_rate):
    """Two policies with different pb_c_init alternate on the default stream with read_back=False: each one's set_params
    rewrites the pooled tree's pb_c table while the other's search is still queued (held behind a spin kernel).  The results
    must equal the same calls made one at a time with read_back=True."""
    B, A = 256, 18
    base = _collect_set(A, 90, B)
    m, _, x, mask, noise = base
    import lightzero_b200 as lzb
    pols = [lzb.MuZeroCollectPolicy(m, dict(num_simulations=30, deterministic=True, discount_factor=DISCOUNT, pb_c_init=c))
            for c in (1.25, 2.5)]

    def once(pol, read_back):
        r = pol.search_batch(x, mask, noise, read_back=read_back, select=(1.0, True, 0))
        return {k: _host(v.clone()) for k, v in r.items()} if read_back else {k: v.clone() for k, v in r.items()}
    ref = [once(p, True) for p in pols]
    assert not np.array_equal(ref[0]["visits"], ref[1]["visits"]), "the two pb_c_init values must lead to different searches"
    torch.cuda.synchronize()
    torch.cuda._sleep(int(0.2 * sleep_rate))
    got = [once(p, False) for p in pols + pols]
    torch.cuda.synchronize()
    for i, g in enumerate(got):
        _same_bits({k: _host(v) for k, v in g.items()}, ref[i % 2], "call %d" % i)
