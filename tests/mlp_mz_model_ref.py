"""The MuZeroModelMLP configs that run on the tensor-core MLP kernel (csrc/mlp_tc.cu, model kind 4), restated by
oracle.model_ref.MuZeroModelMLPRef (lzero/model/muzero_model_mlp.py:21-442 in eval mode: one_hot actions, categorical
supports, norm_type='BN', state_norm=False, no SSL heads).  tests/golden/make_mlp_mz_golden.py pins the restatement bit for
bit to the reference class; the CUDA model is checked against both."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle.model_ref import MuZeroModelMLPRef, emulate_trained_mlp_  # noqa: E402

# name -> (observation_shape, action_space_size, latent_state_dim, res_connection_in_dynamics, head hidden, support range)
CONFIGS = {
    # zoo/box2d/lunarlander/config/lunarlander_disc_muzero_config.py and lunarlander_disc_rezero_mz_config.py
    "lunarlander": (8, 4, 256, True, 32, (-300., 301., 1.)),
    # a latent that is a multiple of 32 but wider than the fp32 kernels' 128, an observation wider than their 160
    "l160_a18": (200, 18, 160, False, 32, (-300., 301., 1.)),
    # a wide observation, narrow head hidden layers and a small support
    "l224_wide": (1000, 64, 224, True, 16, (-10., 11., 1.)),
    # the longest recurrent program: 4 dense dynamics layers, the reward head, 2 prediction layers and the value and policy heads,
    # with 608 support bins and 608 actions cut into 19 FC2 pieces each at L = 32: 66 layers, the kernel's limit
    "l32_a608": (8, 608, 32, True, 32, (-304., 304., 1.)),
    # the widest observation and head hidden layers of a single unit
    "l96_o4096_h1": (4096, 6, 96, False, 1, (-300., 301., 1.)),
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
