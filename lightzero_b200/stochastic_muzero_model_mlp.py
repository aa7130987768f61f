"""Host-side mirror of ``lzero.model.stochastic_muzero_model_mlp.StochasticMuZeroModelMLP`` (the vector-observation Stochastic
MuZero model of the cartpole, lunarlander_disc and pendulum_cont_disc configs).  Same constructor keywords,
``initial_inference(obs)``, ``recurrent_inference(state, option, afterstate=False)`` (stochastic_muzero_model.py:233-273) and
``MZNetworkOutput``; weights from the reference ``state_dict`` (the training-only ``chance_encoder`` and SSL projection
entries are ignored).  Every network runs on the tensor-core kernel of csrc/mlp_tc.cu (math modes tc3 / tc1, ``set_math``),
and the same object plugs into ``StochasticMuZeroMCTSCtree.search`` (one fused CUDA graph).  Inference only (eval mode)."""
from typing import Optional, Sequence

import torch

from . import cabi
from .model_base import StochasticLzModel


class StochasticMuZeroModelMLP(StochasticLzModel):
    _align_latents = True

    def __init__(self, observation_shape: int = 2, action_space_size: int = 6, chance_space_size: int = 2,
                 latent_state_dim: int = 256, reward_head_hidden_channels: Sequence[int] = (32,),
                 value_head_hidden_channels: Sequence[int] = (32,), policy_head_hidden_channels: Sequence[int] = (32,),
                 reward_support_range: Sequence[float] = (-300., 301., 1.),
                 value_support_range: Sequence[float] = (-300., 301., 1.),
                 proj_hid: int = 1024, proj_out: int = 1024, pred_hid: int = 512, pred_out: int = 1024,
                 self_supervised_learning_loss: bool = False, categorical_distribution: bool = True, activation=None,
                 last_linear_layer_init_zero: bool = True, state_norm: bool = False,
                 discrete_action_encoding_type: str = "one_hot", norm_type: Optional[str] = "BN",
                 res_connection_in_dynamics: bool = False, device: Optional[torch.device] = None, **kwargs):
        # proj_* / pred_* / self_supervised_learning_loss shape the training-only SSL heads, last_linear_layer_init_zero the
        # initialisation, and activation is the ReLU the reference's MLP blocks use: all accepted, unused
        if not categorical_distribution or norm_type != "BN" or discrete_action_encoding_type != "one_hot" or state_norm:
            raise NotImplementedError("CUDA StochasticMuZeroModelMLP: categorical_distribution, norm_type='BN', one_hot action "
                                      "encoding, state_norm=False")
        if tuple(reward_support_range) != tuple(value_support_range):
            raise NotImplementedError("reward and value supports must be equal")
        if len(reward_head_hidden_channels) != 1 or len(value_head_hidden_channels) != 1 or len(policy_head_hidden_channels) != 1:
            raise NotImplementedError("heads use exactly one hidden layer (reference default [32])")
        self.observation_shape = int(observation_shape)
        self.action_space_size = int(action_space_size)
        self.chance_space_size = int(chance_space_size)
        self.latent_state_dim = int(latent_state_dim)
        self._latent = (self.latent_state_dim,)
        cfg = cabi.MlpStochasticConfig(self.observation_shape, self.action_space_size, self.chance_space_size,
                                       self.latent_state_dim, reward_head_hidden_channels[0], value_head_hidden_channels[0],
                                       policy_head_hidden_channels[0], int(bool(res_connection_in_dynamics)),
                                       value_support_range[0], value_support_range[1], value_support_range[2])
        self._create(device, "lz_model_create_mlp_stochastic", cfg, value_support_range)
