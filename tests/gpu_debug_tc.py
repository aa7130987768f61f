"""Bring-up diagnostics for the tensor-core (wgmma) path (run on the GPU box; not a pytest).  Single-layer
programs first (localise descriptor / epilogue bugs), then the full network in tc3 and tc1 against
the PyTorch oracle."""
import ctypes
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import lightzero_b200 as lzb
from lightzero_b200 import cabi
from oracle.model_ref import MuZeroModelRef, emulate_trained_

LF_RES, LF_STORE, LF_WRITE, LF_ABIAS, LF_HREW, LF_HVP = 1, 2, 4, 8, 16, 32


def stats(name, got, exp):
    d = (got - exp).abs()
    print(f"{name:28s} max|err| {d.max().item():.3e}  mean|err| {d.mean().item():.3e}  max|exp| {exp.abs().max().item():.3e}")
    return d


def main():
    A, B = 6, int(os.environ.get("DBG_B", 9))
    torch.manual_seed(0)
    ref = emulate_trained_(MuZeroModelRef((4, 84, 84), A), 0)
    cu = lzb.MuZeroModel(observation_shape=(4, 84, 84), action_space_size=A).load_state_dict(ref.state_dict())
    lib = cabi.load()
    g = torch.Generator().manual_seed(1)
    latent = torch.rand(B, 64, 6, 6, generator=g) * 2
    action = torch.randint(0, A, (B,), generator=g)

    def program(layers, flags):
        lw = (ctypes.c_int * len(layers))(*layers)
        lf = (ctypes.c_int * len(layers))(*flags)
        cabi.check(lib.lz_model_debug_tc_program(cu._h, 0, len(layers), lw, lf, 1), "debug program")

    dyn = ref.dynamics_network
    with torch.no_grad():
        onehot = torch.zeros(B, A).scatter_(1, action[:, None], 1)[:, :, None, None].expand(B, A, 6, 6)
        x0 = torch.cat((latent, onehot), 1)
        exp_l0 = torch.relu(dyn.norm_common(dyn.conv(x0)) + latent)
        rb = dyn.resblocks[0]
        exp_c1 = rb.conv1(latent)          # relu(bn(conv(x)))
    for variant in (0,):
        print(f"==== descriptor variant {variant} ====")
        cu.set_math("tc3")
        try:
            program([0], [LF_RES | LF_ABIAS | LF_WRITE | LF_HREW | LF_HVP])
            out = cu.recurrent_inference(latent.cuda(), action.cuda())
            torch.cuda.synchronize()
            d = stats("L0 dyn conv (3 pass)", out.latent_state.cpu(), exp_l0)
            print("  per-pixel mean|err| (6x6):\n", np.array2string(d.mean((0, 1)).numpy(), precision=2))
            program([1], [LF_WRITE | LF_HREW | LF_HVP])
            out = cu.recurrent_inference(latent.cuda(), action.cuda())
            torch.cuda.synchronize()
            d = stats("conv1 of dyn resblock", out.latent_state.cpu(), exp_c1)
            print("  per-pixel mean|err| (6x6):\n", np.array2string(d.mean((0, 1)).numpy(), precision=2))
            print("  per-root max|err|:", d.amax((1, 2, 3)).numpy())
        except Exception as e:
            print("variant", variant, "FAILED:", repr(e))
            return
    # full network
    cu2 = lzb.MuZeroModel(observation_shape=(4, 84, 84), action_space_size=A).load_state_dict(ref.state_dict())
    with torch.no_grad():
        exp = ref.recurrent_inference(latent, action)
    for mode in ("tc3", "tc1"):
        cu2.set_math(mode)
        out = cu2.recurrent_inference(latent.cuda(), action.cuda(), return_scalars=True)
        torch.cuda.synchronize()
        print(f"---- full recurrent_inference, math={mode}")
        stats("next latent", out.latent_state.cpu(), exp.latent_state)
        stats("reward logits", out.reward.cpu(), exp.reward)
        stats("value logits", out.value.cpu(), exp.value)
        stats("policy logits", out.policy_logits.cpu(), exp.policy_logits)
    obs = torch.rand(B, 4, 84, 84, generator=g)
    with torch.no_grad():
        e0 = ref.initial_inference(obs)
    for mode in ("tc3", "tc1"):
        cu2.set_math(mode)
        o = cu2.initial_inference(obs.cuda())
        torch.cuda.synchronize()
        print(f"---- initial_inference, math={mode}")
        stats("latent", o.latent_state.cpu(), e0.latent_state)
        stats("value logits", o.value.cpu(), e0.value)
        stats("policy logits", o.policy_logits.cpu(), e0.policy_logits)
    # timing at the bench size
    Bb = 1024
    lat = torch.rand(Bb, 64, 6, 6).cuda()
    act = torch.randint(0, A, (Bb,)).cuda()
    for mode in ("tc3", "tc1"):
        cu2.set_math(mode)
        for _ in range(3):
            cu2.recurrent_inference(lat, act)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(20):
            cu2.recurrent_inference(lat, act)
        b.record()
        torch.cuda.synchronize()
        print(f"recurrent_inference B=1024 math={mode}: {a.elapsed_time(b) / 20 * 1e3:.1f} us per call (incl. logits outputs + torch allocs)")


if __name__ == "__main__" and not os.environ.get("DBG_PHASES"):
    main()


def phase_breakdown():
    """clock64 stamps of CTA 0 (env LZ_TC_DEBUG=1): where does a k_net_tc launch spend its cycles?"""
    os.environ["LZ_TC_DEBUG"] = "1"
    A = 6
    torch.manual_seed(0)
    ref = emulate_trained_(MuZeroModelRef((4, 84, 84), A), 0)
    cu = lzb.MuZeroModel(observation_shape=(4, 84, 84), action_space_size=A).load_state_dict(ref.state_dict())
    lib = cabi.load()
    lat = torch.rand(1024, 64, 6, 6).cuda()
    act = torch.randint(0, A, (1024,)).cuda()
    for mode in ("tc3", "tc1"):
        cu.set_math(mode)
        for _ in range(3):
            cu.recurrent_inference(lat, act)
        torch.cuda.synchronize()
        buf = (ctypes.c_ulonglong * 64)()
        cabi.check(lib.lz_debug_tc_stamps(buf), "stamps")
        s = list(buf)
        t0 = s[0]
        print(f"== phase breakdown, math={mode} (cycles since epilogue start)")
        print(f"   load done            {s[1] - t0:8d}")
        for L in range(5):
            print(f"   L{L}: mma issue {s[32 + 2 * L] - t0:8d} -> {s[33 + 2 * L] - t0:8d} | acc ready {s[2 + 2 * L] - t0:8d}  epilogue done {s[3 + 2 * L] - t0:8d}")
        print(f"   early reward head done {s[28] - t0:8d}   (runs under the next layer's MMAs)")
        print(f"   hooks ready            {s[24] - t0:8d}")
        print(f"   heads + outputs done   {s[27] - t0:8d}")


if __name__ == "__main__" and os.environ.get("DBG_PHASES"):
    phase_breakdown()
