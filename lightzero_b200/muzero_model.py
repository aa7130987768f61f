"""Host-side mirror of ``lzero.model.muzero_model.MuZeroModel`` (muzero_model.py:20-272): same
constructor keywords, ``initial_inference`` / ``recurrent_inference`` with the same argument meaning
and the same ``MZNetworkOutput``, weights ingested from the reference ``state_dict`` key layout.
The forward passes are the fused CUDA kernels behind ``lz_model_*`` (include/lzb200.h); there is no
PyTorch eager path.  Inference (eval mode, BatchNorm running statistics) only.
"""
from dataclasses import dataclass
from typing import Dict, Optional, Sequence

import itertools

import torch

from . import cabi

_model_serial = itertools.count(1)      # never reused (unlike id()): keys of the per-tree lz_search caches in mz_tree


@dataclass
class MZNetworkOutput:
    """lzero/model/common.py:131-141"""
    value: torch.Tensor
    reward: torch.Tensor
    policy_logits: torch.Tensor
    latent_state: torch.Tensor


class MuZeroModel:
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
        if not torch.cuda.is_available():
            raise RuntimeError("lightzero_b200.MuZeroModel needs a CUDA device; there is no CPU fallback")
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.observation_shape = tuple(observation_shape)
        self.action_space_size = action_space_size
        self.num_channels = num_channels
        self._lib = cabi.load()
        cfg = cabi.ModelConfig(observation_shape[0], observation_shape[1], observation_shape[2], action_space_size,
                               num_res_blocks, num_channels, reward_head_channels, value_head_channels,
                               policy_head_channels, reward_head_hidden_channels[0], value_head_hidden_channels[0],
                               policy_head_hidden_channels[0], value_support_range[0], value_support_range[1],
                               value_support_range[2], int(efficientzero),
                               int(kwargs.get("lstm_hidden_size", 0) if efficientzero else 0), int(bool(downsample)))
        self._cfg = cfg
        h = cabi.c_void_p()
        with torch.cuda.device(self.device):
            cabi.check(self._lib.lz_model_create(cfg, h), "lz_model_create")
        self._h = h
        self._serial = next(_model_serial)
        self.latent_hw = self._lib.lz_model_latent_hw(self._h)
        shape = (cabi.ctypes.c_int32 * 3)()
        cabi.check(self._lib.lz_model_latent_shape(self._h, cabi.ctypes.byref(shape, 0), cabi.ctypes.byref(shape, 4),
                                                   cabi.ctypes.byref(shape, 8)), "lz_model_latent_shape")
        self.latent_shape = tuple(shape)          # (C, H, W) of one root's latent
        self.downsample = bool(downsample)
        self.value_support_size = self.reward_support_size = self._lib.lz_model_support_size(self._h)
        self._loaded = False

    # ---- weights -------------------------------------------------------------------------------
    def load_state_dict(self, state_dict: Dict[str, torch.Tensor], strict: bool = True):
        """Takes a reference ``MuZeroModel.state_dict()`` (SURVEY.md App. B.4 key layout)."""
        with torch.cuda.device(self.device):
            for name, t in state_dict.items():
                if not torch.is_floating_point(t):
                    continue
                a = t.detach().to("cpu", torch.float32).contiguous()
                cabi.check(self._lib.lz_model_set_tensor(self._h, name.encode(), a.data_ptr(), a.numel()),
                           "lz_model_set_tensor")
            cabi.check(self._lib.lz_model_finalize(self._h), "lz_model_finalize")
        self._loaded = True
        return self

    @classmethod
    def from_state_dict(cls, state_dict, **cfg):
        return cls(**cfg).load_state_dict(state_dict)

    MATH_MODES = {"tc3": 1, "tc1": 2}

    def set_math(self, mode):
        """'tc3' = wgmma 3xFP16 (fp32-accurate, the default), 'tc1' = wgmma single fp16 pass."""
        if isinstance(mode, str) and mode not in self.MATH_MODES:
            raise ValueError(f"set_math: unknown mode {mode!r}: the conv models run tc3 or tc1")
        code = self.MATH_MODES[mode] if isinstance(mode, str) else int(mode)
        cabi.check(self._lib.lz_model_set_math(self._h, code), "lz_model_set_math")
        self.math = code
        return self

    def eval(self):
        return self

    def to(self, *a, **k):
        return self

    # ---- forward -------------------------------------------------------------------------------
    def _check(self):
        if not self._loaded:
            raise RuntimeError("MuZeroModel: load_state_dict() has not been called")

    def initial_inference(self, obs: torch.Tensor, return_scalar_value: bool = False) -> MZNetworkOutput:
        """muzero_model.py:210-240.  ``reward`` is the python list of zeros the reference returns."""
        self._check()
        obs = obs.to(self.device, torch.float32).contiguous()
        B = obs.shape[0]
        latent = torch.empty((B,) + self.latent_shape, device=self.device)
        policy = torch.empty(B, self.action_space_size, device=self.device)
        value = torch.empty(B, self.value_support_size, device=self.device)
        scalar = torch.empty(B, device=self.device) if return_scalar_value else None
        with torch.cuda.device(self.device):
            cabi.check(self._lib.lz_model_initial_inference(self._h, B, obs.data_ptr(), latent.data_ptr(),
                                                            policy.data_ptr(), value.data_ptr(), cabi.ptr(scalar),
                                                            cabi.stream_ptr()), "lz_model_initial_inference")
        out = MZNetworkOutput(value, [0. for _ in range(B)], policy, latent)
        if return_scalar_value:
            out.value_scalar = scalar
        return out

    def recurrent_inference(self, latent_state: torch.Tensor, action: torch.Tensor,
                            return_scalars: bool = False) -> MZNetworkOutput:
        """muzero_model.py:242-272; ``action`` is (B,) or (B,1) integer."""
        self._check()
        latent_state = latent_state.to(self.device, torch.float32).contiguous()
        action = action.to(self.device).reshape(-1).to(torch.int32).contiguous()
        B = latent_state.shape[0]
        nxt = torch.empty((B,) + self.latent_shape, device=self.device)
        policy = torch.empty(B, self.action_space_size, device=self.device)
        value = torch.empty(B, self.value_support_size, device=self.device)
        reward = torch.empty(B, self.reward_support_size, device=self.device)
        rs = torch.empty(B, device=self.device) if return_scalars else None
        vs = torch.empty(B, device=self.device) if return_scalars else None
        with torch.cuda.device(self.device):
            cabi.check(self._lib.lz_model_recurrent_inference(
                self._h, B, latent_state.data_ptr(), action.data_ptr(), nxt.data_ptr(), reward.data_ptr(),
                value.data_ptr(), policy.data_ptr(), cabi.ptr(rs), cabi.ptr(vs), cabi.stream_ptr()),
                "lz_model_recurrent_inference")
        out = MZNetworkOutput(value, reward, policy, nxt)
        if return_scalars:
            out.reward_scalar, out.value_scalar = rs, vs
        return out

    def inverse_scalar_transform(self, logits: torch.Tensor) -> torch.Tensor:
        logits = logits.to(self.device, torch.float32).contiguous()
        out = torch.empty(logits.shape[0], 1, device=self.device)
        with torch.cuda.device(self.device):
            cabi.check(self._lib.lz_inverse_scalar_transform(self._h, logits.shape[0], logits.data_ptr(),
                                                             out.data_ptr(), cabi.stream_ptr()),
                       "lz_inverse_scalar_transform")
        return out

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                from . import mz_tree
                mz_tree.drop_model_searches(self._serial)     # lz_search handles point at this lz_model: destroy them first
                self._lib.lz_model_destroy(self._h)
        except Exception:
            pass
