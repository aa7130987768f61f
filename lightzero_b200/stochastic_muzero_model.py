"""Host-side mirror of ``lzero.model.stochastic_muzero_model.StochasticMuZeroModel`` with ``downsample=False`` (the board
network of the 2048 config).  Same constructor keywords, ``initial_inference(obs)``,
``recurrent_inference(state, option, afterstate=False)`` (stochastic_muzero_model.py:233-273) and ``MZNetworkOutput``; latents
are (B, num_channels, H, W).  Weights come from the reference ``state_dict`` (the training-only ``chance_encoder`` and SSL
projection entries are ignored).  Every program runs on the board tensor-core kernel of csrc/board_tc.cu (math modes tc3 / tc1,
``set_math``), and the same object plugs into ``StochasticMuZeroMCTSCtree.search`` and ``StochasticMuZeroCollectPolicy`` (one
fused CUDA graph each).  Inference only (eval mode)."""
from typing import Optional, Sequence

import torch

from . import cabi
from .model_base import StochasticLzModel


class StochasticMuZeroModel(StochasticLzModel):
    def __init__(self, observation_shape: Sequence[int] = (12, 96, 96), action_space_size: int = 6,
                 chance_space_size: int = 2, num_res_blocks: int = 1, num_channels: int = 64, reward_head_channels: int = 16,
                 value_head_channels: int = 16, policy_head_channels: int = 16,
                 reward_head_hidden_channels: Sequence[int] = (32,), value_head_hidden_channels: Sequence[int] = (32,),
                 policy_head_hidden_channels: Sequence[int] = (32,),
                 reward_support_range: Sequence[float] = (-300., 301., 1.),
                 value_support_range: Sequence[float] = (-300., 301., 1.),
                 proj_hid: int = 1024, proj_out: int = 1024, pred_hid: int = 512, pred_out: int = 1024,
                 self_supervised_learning_loss: bool = False, categorical_distribution: bool = True, activation=None,
                 last_linear_layer_init_zero: bool = True, state_norm: bool = False, downsample: bool = False,
                 device: Optional[torch.device] = None, **kwargs):
        # proj_* / pred_* / self_supervised_learning_loss shape the training-only SSL heads, last_linear_layer_init_zero the
        # initialisation, and activation is the ReLU the reference's networks use: all accepted, unused; other keywords are
        # swallowed as the reference's *args / **kwargs are
        if downsample:
            raise NotImplementedError("CUDA StochasticMuZeroModel: downsample=True (the Atari Stochastic MuZero network) is not "
                                      "implemented; the board network (downsample=False) is")
        if not categorical_distribution or state_norm:
            raise NotImplementedError("CUDA StochasticMuZeroModel: categorical_distribution=True and state_norm=False")
        if tuple(reward_support_range) != tuple(value_support_range):
            raise NotImplementedError("reward and value supports must be equal")
        if len(reward_head_hidden_channels) != 1 or len(value_head_hidden_channels) != 1 or len(policy_head_hidden_channels) != 1:
            raise NotImplementedError("heads use exactly one hidden layer (reference default [32])")
        self.observation_shape = tuple(observation_shape)
        self.action_space_size = int(action_space_size)
        self.chance_space_size = int(chance_space_size)
        self.num_channels = int(num_channels)
        base = cabi.ModelConfig(observation_shape[0], observation_shape[1], observation_shape[2], self.action_space_size,
                                num_res_blocks, self.num_channels, reward_head_channels, value_head_channels,
                                policy_head_channels, reward_head_hidden_channels[0], value_head_hidden_channels[0],
                                policy_head_hidden_channels[0], value_support_range[0], value_support_range[1],
                                value_support_range[2], 0, 0, 0)
        self._create(device, "lz_model_create_stochastic", cabi.StochasticConfig(base, self.chance_space_size),
                     value_support_range)
        self.latent_shape = self._latent = (self.num_channels,) + self.observation_shape[1:]
