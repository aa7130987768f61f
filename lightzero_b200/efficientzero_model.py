"""Host-side mirror of ``lzero.model.efficientzero_model.EfficientZeroModel`` (efficientzero_model.py:20-272): same
constructor keywords, ``initial_inference(obs)`` / ``recurrent_inference(latent_state, reward_hidden_state, action)`` with
the same ``EZNetworkOutput``; weights come from the reference ``state_dict`` (the training-only SSL ``projection`` /
``prediction_head`` entries are ignored).  The conv trunk and the prediction heads run on the wgmma kernels shared with
``MuZeroModel``; the value-prefix head (conv1x1 -> BN -> ReLU -> LSTM -> BN -> ReLU -> MLP, :552-569) is a batched GEMM +
fused cell update (csrc/ez.cu).  Inference only (eval mode)."""
from typing import Optional, Sequence

import torch

from .model_base import EZNetworkOutput  # noqa: F401  (part of this module's interface)
from .muzero_model import MuZeroModel


class EfficientZeroModel(MuZeroModel):
    value_prefix = True

    def __init__(self, observation_shape: Sequence[int] = (4, 96, 96), action_space_size: int = 6,
                 lstm_hidden_size: int = 512, downsample: Optional[bool] = None, device: Optional[torch.device] = None, **kwargs):
        kwargs.pop("_efficientzero", None)
        super().__init__(observation_shape=observation_shape, action_space_size=action_space_size, downsample=downsample,
                         device=device, _efficientzero=True, lstm_hidden_size=lstm_hidden_size, **kwargs)
        self.lstm_hidden_size = lstm_hidden_size

    def recurrent_inference(self, latent_state: torch.Tensor, reward_hidden_state, action: torch.Tensor,
                            return_scalars: bool = False) -> EZNetworkOutput:
        """efficientzero_model.py:240-272; ``reward_hidden_state`` is the (1, B, H) pair the reference hands to nn.LSTM."""
        return self._recurrent(latent_state, reward_hidden_state, action, return_scalars)
