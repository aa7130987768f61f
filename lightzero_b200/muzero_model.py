"""Host-side mirror of ``lzero.model.muzero_model.MuZeroModel`` (muzero_model.py:20-272): same
constructor keywords, ``initial_inference`` / ``recurrent_inference`` with the same argument meaning
and the same ``MZNetworkOutput``, weights ingested from the reference ``state_dict`` key layout.
The forward passes are the fused CUDA kernels behind ``lz_model_*`` (include/lzb200.h); there is no
PyTorch eager path.  Inference (eval mode, BatchNorm running statistics) only.
"""
from typing import Optional, Sequence

import torch

from . import cabi
from .model_base import LzModel, MZNetworkOutput  # noqa: F401  (MZNetworkOutput is part of this module's interface)


class MuZeroModel(LzModel):
    def __init__(self, observation_shape: Sequence[int] = (4, 84, 84), action_space_size: int = 6,
                 num_res_blocks: int = 1, num_channels: int = 64, reward_head_channels: int = 16,
                 value_head_channels: int = 16, policy_head_channels: int = 16,
                 reward_head_hidden_channels: Sequence[int] = (32,), value_head_hidden_channels: Sequence[int] = (32,),
                 policy_head_hidden_channels: Sequence[int] = (32,),
                 reward_support_range: Sequence[float] = (-300., 301., 1.),
                 value_support_range: Sequence[float] = (-300., 301., 1.),
                 categorical_distribution: bool = True, downsample: Optional[bool] = None, norm_type: str = "BN",
                 discrete_action_encoding_type: str = "one_hot", state_norm: bool = False,
                 device: Optional[torch.device] = None, **kwargs):
        # unknown kwargs are swallowed like muzero_model.py:49-50
        efficientzero = bool(kwargs.get("_efficientzero", False))
        board = tuple(observation_shape[1:])
        fits_board = len(board) == 2 and 1 <= board[0] <= 8 and 1 <= board[1] <= 8
        if downsample is None:
            # The reference's default is downsample=False (muzero_model.py:45, efficientzero_model.py:45): the full-resolution
            # network of the board-game configs, which this class runs for MuZero boards up to 8x8.  84 / 96-pixel models
            # default to the DownSample network here, as they always have.  A 64x64 model follows the reference default, so
            # it must ask for DownSample as the shipped Atari configs do (zoo/atari/config/atari_muzero_config.py:56,
            # atari_efficientzero_config.py:44).
            downsample = not (fits_board and not efficientzero)
            if board == (64, 64):
                raise NotImplementedError(
                    "a 64x64 observation_shape needs downsample=True (as in the reference's Atari configs): with the reference's "
                    "default downsample=False the model is a full-resolution network, which this CUDA model implements for "
                    "boards up to 8x8 only")
        if not downsample and (efficientzero or not fits_board):
            raise NotImplementedError(
                "downsample=False (the full-resolution board network) is implemented for MuZeroModel on boards up to 8x8; "
                f"got observation_shape {tuple(observation_shape)}" + (" for EfficientZeroModel" if efficientzero else ""))
        if not categorical_distribution or norm_type != "BN" or discrete_action_encoding_type != "one_hot" or state_norm:
            raise NotImplementedError(
                "CUDA MuZeroModel implements the configurations of the reference's Atari and board-game configs: "
                "categorical_distribution, norm_type='BN', one_hot action encoding, state_norm=False")
        if tuple(reward_support_range) != tuple(value_support_range):
            raise NotImplementedError("reward and value supports must be equal")
        if len(reward_head_hidden_channels) != 1 or len(value_head_hidden_channels) != 1 or len(policy_head_hidden_channels) != 1:
            raise NotImplementedError("heads use exactly one hidden layer (reference default [32])")
        self.observation_shape = tuple(observation_shape)
        self.action_space_size = action_space_size
        self.num_channels = num_channels
        cfg = cabi.ModelConfig(observation_shape[0], observation_shape[1], observation_shape[2], action_space_size,
                               num_res_blocks, num_channels, reward_head_channels, value_head_channels,
                               policy_head_channels, reward_head_hidden_channels[0], value_head_hidden_channels[0],
                               policy_head_hidden_channels[0], value_support_range[0], value_support_range[1],
                               value_support_range[2], int(efficientzero),
                               int(kwargs.get("lstm_hidden_size", 0) if efficientzero else 0), int(bool(downsample)))
        self._cfg = cfg
        self._create(device, "lz_model_create", cfg, value_support_range)
        self.latent_hw = self._lib.lz_model_latent_hw(self._h)
        shape = (cabi.ctypes.c_int32 * 3)()
        cabi.check(self._lib.lz_model_latent_shape(self._h, cabi.ctypes.byref(shape, 0), cabi.ctypes.byref(shape, 4),
                                                   cabi.ctypes.byref(shape, 8)), "lz_model_latent_shape")
        self.latent_shape = self._latent = tuple(shape)          # (C, H, W) of one root's latent
        self.downsample = bool(downsample)

    @classmethod
    def from_state_dict(cls, state_dict, **cfg):
        return cls(**cfg).load_state_dict(state_dict)

    def inverse_scalar_transform(self, logits: torch.Tensor) -> torch.Tensor:
        logits = logits.to(self.device, torch.float32).contiguous()
        out = torch.empty(logits.shape[0], 1, device=self.device)
        with torch.cuda.device(self.device):
            cabi.check(self._lib.lz_inverse_scalar_transform(self._h, logits.shape[0], logits.data_ptr(),
                                                             out.data_ptr(), cabi.stream_ptr()),
                       "lz_inverse_scalar_transform")
        return out
