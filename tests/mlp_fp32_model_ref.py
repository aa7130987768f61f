"""The MuZeroModelMLP configs that run on the fp32 MLP kernels (csrc/mlp.cu, model kind 1), restated by
oracle.model_ref.MuZeroModelMLPRef (lzero/model/muzero_model_mlp.py:21-442 in eval mode: one_hot actions, categorical
supports, norm_type='BN', state_norm=False).  tests/golden/make_mlp_fp32_golden.py pins the restatement bit for bit to the
reference class; the CUDA model is checked against both.

The shipped rows are the reference's vector-observation MuZero configs; the edge rows sit on the borders of the fp32
kernels' envelope (latent in [8, 128], obs <= 160, latent + A <= 160, head hidden <= 160, support size <= 608).  Between
them the input counts of the dense layers (obs, latent, head hidden) take every remainder mod 8, so the clamped tail of
the kernel's 8-wide input loop runs at every length."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle.model_ref import MuZeroModelMLPRef, emulate_trained_mlp_  # noqa: E402

SUPPORT = (-300., 301., 1.)

# name -> (observation_shape, action_space_size, latent_state_dim, res_connection_in_dynamics, head hidden, support range)
CONFIGS = {
    # zoo/classic_control/cartpole/config/cartpole_{muzero,rezero_mz,gumbel_muzero}_config.py, with the residual dynamics
    # of the ReZero / lunarlander family (tests/test_gpu_mlp.py covers cartpole without it)
    "cartpole": (4, 2, 128, True, 32, SUPPORT),
    # zoo/classic_control/mountain_car/config/mountain_car_muzero_config.py
    "mountain_car": (2, 3, 64, False, 32, SUPPORT),
    # zoo/classic_control/pendulum/config/pendulum_cont_disc_{muzero,gumbel_muzero}_config.py
    "pendulum": (3, 11, 128, False, 32, SUPPORT),
    # zoo/bsuite/config/bsuite_muzero_config.py: bandit_noise/0 and bsuite_swingup/0
    "bsuite_bandit": (1, 11, 128, False, 32, SUPPORT),
    "bsuite_swingup": (8, 3, 128, False, 32, SUPPORT),
    # zoo/memory/config/memory_muzero_config.py
    "memory": (25, 4, 128, False, 32, SUPPORT),
    # the narrowest latent with the most actions it allows (latent + A = 160), one-unit head hidden layers, a small support
    "l8_a152": (6, 152, 8, True, 1, (-10., 11., 1.)),
    # the widest observation and head hidden layers, a latent that is not a multiple of 32, the largest support (608 logits)
    "l100_o160": (160, 60, 100, False, 160, (-303., 305., 1.)),
    # the widest latent with 32 actions
    "l128_a32": (25, 32, 128, True, 32, SUPPORT),
    # a half-unit support step (exact in binary), a latent between one and two warps wide
    "l44_half": (15, 7, 44, True, 21, (-20., 20.5, 0.5)),
}


def model_kwargs(name):
    obs, A, L, res, hid, sup = CONFIGS[name]
    return dict(observation_shape=obs, action_space_size=A, latent_state_dim=L, res_connection_in_dynamics=res,
                reward_head_hidden_channels=[hid], value_head_hidden_channels=[hid], policy_head_hidden_channels=[hid],
                reward_support_range=sup, value_support_range=sup)


def build(name, seed, dtype=torch.float32):
    torch.manual_seed(seed)
    return emulate_trained_mlp_(MuZeroModelMLPRef(**model_kwargs(name)), seed).to(dtype).eval()


def scalar(logits, support):
    """softmax . support -> h^-1 in float64"""
    x = torch.as_tensor(logits).double()
    v = (torch.softmax(x, -1) * torch.arange(*support, dtype=torch.float64)).sum(-1)
    eps = 0.001
    return torch.sign(v) * (((torch.sqrt(1 + 4 * eps * (torch.abs(v) + 1 + eps)) - 1) / (2 * eps)) ** 2 - 1)
