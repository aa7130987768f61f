"""Host-side mirror of ``lzero.model.efficientzero_model.EfficientZeroModel`` (efficientzero_model.py:20-272): same
constructor keywords, ``initial_inference(obs)`` / ``recurrent_inference(latent_state, reward_hidden_state, action)`` with
the same ``EZNetworkOutput``; weights come from the reference ``state_dict`` (the training-only SSL ``projection`` /
``prediction_head`` entries are ignored).  The conv trunk and the prediction heads run on the wgmma kernels shared with
``MuZeroModel``; the value-prefix head (conv1x1 -> BN -> ReLU -> LSTM -> BN -> ReLU -> MLP, :552-569) is a batched GEMM +
fused cell update (csrc/ez.cu).  Inference only (eval mode)."""
from dataclasses import dataclass
from typing import Optional, Sequence, Tuple

import torch

from . import cabi
from .muzero_model import MuZeroModel


@dataclass
class EZNetworkOutput:
    """lzero/model/common.py:119-128"""
    value: torch.Tensor
    value_prefix: torch.Tensor
    policy_logits: torch.Tensor
    latent_state: torch.Tensor
    reward_hidden_state: Tuple[torch.Tensor, torch.Tensor]


class EfficientZeroModel(MuZeroModel):
    def __init__(self, observation_shape: Sequence[int] = (4, 96, 96), action_space_size: int = 6,
                 lstm_hidden_size: int = 512, downsample: Optional[bool] = None, device: Optional[torch.device] = None, **kwargs):
        kwargs.pop("_efficientzero", None)
        super().__init__(observation_shape=observation_shape, action_space_size=action_space_size, downsample=downsample,
                         device=device, _efficientzero=True, lstm_hidden_size=lstm_hidden_size, **kwargs)
        self.lstm_hidden_size = lstm_hidden_size

    MATH_MODES = {"tc3": 1, "tc1": 2}

    def initial_inference(self, obs: torch.Tensor, return_scalar_value: bool = False) -> EZNetworkOutput:
        """efficientzero_model.py:203-238: value / policy / latent as MuZero, zero (1, B, H) reward hidden state."""
        o = super().initial_inference(obs, return_scalar_value)
        B = o.latent_state.shape[0]
        hidden = (torch.zeros(1, B, self.lstm_hidden_size, device=self.device), torch.zeros(1, B, self.lstm_hidden_size, device=self.device))
        out = EZNetworkOutput(o.value, [0. for _ in range(B)], o.policy_logits, o.latent_state, hidden)
        if return_scalar_value:
            out.value_scalar = o.value_scalar
        return out

    def recurrent_inference(self, latent_state: torch.Tensor, reward_hidden_state, action: torch.Tensor,
                            return_scalars: bool = False) -> EZNetworkOutput:
        """efficientzero_model.py:240-272; ``reward_hidden_state`` is the (1, B, H) pair the reference hands to nn.LSTM."""
        self._check()
        latent_state = latent_state.to(self.device, torch.float32).contiguous()
        action = action.to(self.device).reshape(-1).to(torch.int32).contiguous()
        B, hw, C, H = latent_state.shape[0], self.latent_hw, self.num_channels, self.lstm_hidden_size
        h0 = reward_hidden_state[0].to(self.device, torch.float32).reshape(B, H).contiguous()
        h1 = reward_hidden_state[1].to(self.device, torch.float32).reshape(B, H).contiguous()
        nxt = torch.empty(B, C, hw, hw, device=self.device)
        n0, n1 = torch.empty(1, B, H, device=self.device), torch.empty(1, B, H, device=self.device)
        policy = torch.empty(B, self.action_space_size, device=self.device)
        value = torch.empty(B, self.value_support_size, device=self.device)
        vprefix = torch.empty(B, self.reward_support_size, device=self.device)
        ps = torch.empty(B, device=self.device) if return_scalars else None
        vs = torch.empty(B, device=self.device) if return_scalars else None
        with torch.cuda.device(self.device):
            cabi.check(self._lib.lz_model_recurrent_inference_ez(
                self._h, B, latent_state.data_ptr(), h0.data_ptr(), h1.data_ptr(), action.data_ptr(), nxt.data_ptr(),
                n0.data_ptr(), n1.data_ptr(), vprefix.data_ptr(), value.data_ptr(), policy.data_ptr(), cabi.ptr(ps),
                cabi.ptr(vs), cabi.stream_ptr()), "lz_model_recurrent_inference_ez")
        out = EZNetworkOutput(value, vprefix, policy, nxt, (n0, n1))
        if return_scalars:
            out.value_prefix_scalar, out.value_scalar = ps, vs
        return out
