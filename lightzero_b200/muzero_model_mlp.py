"""Host-side mirror of ``lzero.model.muzero_model_mlp.MuZeroModelMLP`` (muzero_model_mlp.py:21-295):
vector observations (BASELINE config 1: CartPole, obs 4, latent 128, A=2; lunarlander and its ReZero variant, latent 256).
Same constructor keywords, ``initial_inference`` / ``recurrent_inference`` and ``MZNetworkOutput``; weights from the
reference ``state_dict``.  The library picks the kernels from the config: the fp32 kernels of csrc/mlp.cu take latents up to
128 with obs_dim and latent + actions up to 160; every other config with a latent that is a multiple of 32 up to 256 runs on
the tensor-core kernel of csrc/mlp_tc.cu (math modes tc3 / tc1, ``set_math``).  The same object plugs into
``MuZeroMCTSCtree.search`` / ``search_with_reuse``, ``GumbelMuZeroMCTSCtree.search``, ``MuZeroCollectPolicy`` and reanalyze
like the conv model."""
from typing import Optional, Sequence

import torch

from . import cabi
from .model_base import LzModel


class MuZeroModelMLP(LzModel):
    _align_latents = True

    def __init__(self, observation_shape: int = 4, action_space_size: int = 2, latent_state_dim: int = 128,
                 reward_head_hidden_channels: Sequence[int] = (32,), value_head_hidden_channels: Sequence[int] = (32,),
                 policy_head_hidden_channels: Sequence[int] = (32,),
                 reward_support_range: Sequence[float] = (-300., 301., 1.),
                 value_support_range: Sequence[float] = (-300., 301., 1.),
                 categorical_distribution: bool = True, norm_type: str = "BN",
                 discrete_action_encoding_type: str = "one_hot", state_norm: bool = False,
                 res_connection_in_dynamics: bool = False, device: Optional[torch.device] = None, **kwargs):
        if not categorical_distribution or norm_type != "BN" or discrete_action_encoding_type != "one_hot" or state_norm:
            raise NotImplementedError("CUDA MuZeroModelMLP: categorical_distribution, norm_type='BN', one_hot, state_norm=False")
        if tuple(reward_support_range) != tuple(value_support_range):
            raise NotImplementedError("reward and value supports must be equal")
        self.observation_shape = int(observation_shape)
        self.action_space_size = action_space_size
        self.latent_state_dim = latent_state_dim
        self._latent = (latent_state_dim,)
        cfg = cabi.MlpConfig(self.observation_shape, action_space_size, latent_state_dim, reward_head_hidden_channels[0],
                             value_head_hidden_channels[0], policy_head_hidden_channels[0], int(bool(res_connection_in_dynamics)),
                             value_support_range[0], value_support_range[1], value_support_range[2])
        self._create(device, "lz_model_create_mlp", cfg, value_support_range)
