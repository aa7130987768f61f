"""Host-side mirror of ``lzero.model.efficientzero_model_mlp.EfficientZeroModelMLP`` (efficientzero_model_mlp.py:16-300): the
EfficientZero model of the reference's vector-observation configs (cartpole, lunarlander, bipedalwalker, minigrid, pendulum, memory,
bsuite).  Same constructor keywords and defaults, ``initial_inference(obs)`` / ``recurrent_inference(latent_state,
reward_hidden_state, action)`` and ``EZNetworkOutput``; weights from the reference ``state_dict`` (the training-only SSL
``projection`` / ``prediction_head`` entries are ignored).  The dense layers run on the wgmma kernel of csrc/mlp_tc.cu, the
LSTM value-prefix head on ez.cu's; the same object plugs into ``EfficientZeroMCTSCtree.search`` / ``search_with_reuse``
(fused one-graph searches), ``EfficientZeroCollectPolicy`` and the EfficientZero reanalyze.  Inference only (eval mode)."""
from typing import Optional, Sequence

import torch

from . import cabi
from .model_base import EZNetworkOutput, LzModel


class EfficientZeroModelMLP(LzModel):
    value_prefix = True
    _align_latents = True

    def __init__(self, observation_shape: int = 2, action_space_size: int = 6, lstm_hidden_size: int = 512,
                 latent_state_dim: int = 256, reward_head_hidden_channels: Sequence[int] = (32,),
                 value_head_hidden_channels: Sequence[int] = (32,), policy_head_hidden_channels: Sequence[int] = (32,),
                 reward_support_range: Sequence[float] = (-300., 301., 1.),
                 value_support_range: Sequence[float] = (-300., 301., 1.),
                 proj_hid: int = 1024, proj_out: int = 1024, pred_hid: int = 512, pred_out: int = 1024,
                 self_supervised_learning_loss: bool = True, categorical_distribution: bool = True,
                 last_linear_layer_init_zero: bool = True, state_norm: bool = False, activation=None,
                 norm_type: Optional[str] = "BN", discrete_action_encoding_type: str = "one_hot",
                 res_connection_in_dynamics: bool = False, device: Optional[torch.device] = None, **kwargs):
        # proj_* / pred_* / self_supervised_learning_loss shape the training-only SSL heads; last_linear_layer_init_zero and
        # activation only shape the initialisation / the dynamics activation the reference fixes to ReLU: all accepted, unused
        if not categorical_distribution or norm_type != "BN" or discrete_action_encoding_type != "one_hot" or state_norm:
            raise NotImplementedError("CUDA EfficientZeroModelMLP: categorical_distribution, norm_type='BN', one_hot action "
                                      "encoding, state_norm=False")
        if tuple(reward_support_range) != tuple(value_support_range):
            raise NotImplementedError("reward and value supports must be equal")
        if len(reward_head_hidden_channels) != 1 or len(value_head_hidden_channels) != 1 or len(policy_head_hidden_channels) != 1:
            raise NotImplementedError("heads use exactly one hidden layer (reference default [32])")
        self.observation_shape = int(observation_shape)
        self.action_space_size = int(action_space_size)
        self.latent_state_dim = int(latent_state_dim)
        self.lstm_hidden_size = int(lstm_hidden_size)
        self._latent = (self.latent_state_dim,)
        cfg = cabi.MlpEzConfig(self.observation_shape, self.action_space_size, self.latent_state_dim, self.lstm_hidden_size,
                               reward_head_hidden_channels[0], value_head_hidden_channels[0], policy_head_hidden_channels[0],
                               int(bool(res_connection_in_dynamics)), value_support_range[0], value_support_range[1],
                               value_support_range[2])
        self._create(device, "lz_model_create_mlp_ez", cfg, value_support_range)

    def recurrent_inference(self, latent_state: torch.Tensor, reward_hidden_state, action: torch.Tensor,
                            return_scalars: bool = False) -> EZNetworkOutput:
        """efficientzero_model_mlp.py:187-300; ``reward_hidden_state`` is the (1, B, H) pair the reference hands to nn.LSTM."""
        return self._recurrent(latent_state, reward_hidden_state, action, return_scalars)
