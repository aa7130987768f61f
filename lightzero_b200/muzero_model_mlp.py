"""Host-side mirror of ``lzero.model.muzero_model_mlp.MuZeroModelMLP`` (muzero_model_mlp.py:21-295):
vector observations (BASELINE config 1: CartPole, obs 4, latent 128, A=2; lunarlander and its ReZero variant, latent 256).
Same constructor keywords, ``initial_inference`` / ``recurrent_inference`` and ``MZNetworkOutput``; weights from the
reference ``state_dict``.  The library picks the kernels from the config: the fp32 kernels of csrc/mlp.cu take latents up to
128 with obs_dim and latent + actions up to 160; every other config with a latent that is a multiple of 32 up to 256 runs on
the tensor-core kernel of csrc/mlp_tc.cu (math modes tc3 / tc1, ``set_math``).  The same object plugs into
``MuZeroMCTSCtree.search`` / ``search_with_reuse``, ``GumbelMuZeroMCTSCtree.search``, ``MuZeroCollectPolicy`` and reanalyze
like the conv model."""
from typing import Dict, Optional, Sequence

import torch

from . import cabi
from .muzero_model import MZNetworkOutput


class MuZeroModelMLP:
    MATH_MODES = {"tc3": 1, "tc1": 2}

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
        if not torch.cuda.is_available():
            raise RuntimeError("lightzero_b200.MuZeroModelMLP needs a CUDA device; there is no CPU fallback")
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.observation_shape = int(observation_shape)
        self.action_space_size = action_space_size
        self.latent_state_dim = latent_state_dim
        self._lib = cabi.load()
        cfg = cabi.MlpConfig(self.observation_shape, action_space_size, latent_state_dim, reward_head_hidden_channels[0],
                             value_head_hidden_channels[0], policy_head_hidden_channels[0], int(bool(res_connection_in_dynamics)),
                             value_support_range[0], value_support_range[1], value_support_range[2])
        h = cabi.c_void_p()
        with torch.cuda.device(self.device):
            cabi.check(self._lib.lz_model_create_mlp(cfg, h), "lz_model_create_mlp")
        self._h = h
        from .muzero_model import _model_serial
        self._serial = next(_model_serial)      # key of the per-tree lz_search caches (mz_tree)
        self.value_support_size = self.reward_support_size = self._lib.lz_model_support_size(self._h)
        self._loaded = False

    def load_state_dict(self, state_dict: Dict[str, torch.Tensor], strict: bool = True):
        with torch.cuda.device(self.device):
            for name, t in state_dict.items():
                if not torch.is_floating_point(t):
                    continue
                a = t.detach().to("cpu", torch.float32).contiguous()
                cabi.check(self._lib.lz_model_set_tensor(self._h, name.encode(), a.data_ptr(), a.numel()), "lz_model_set_tensor")
            cabi.check(self._lib.lz_model_finalize(self._h), "lz_model_finalize")
        self._loaded = True
        return self

    def set_math(self, mode):
        """'tc3' = wgmma 3xFP16 (fp32-accurate, the default), 'tc1' = wgmma single fp16 pass.  Tensor-core configs only: a
        model on the fp32 kernels has no math mode (LzError)."""
        if isinstance(mode, str) and mode not in self.MATH_MODES:
            raise ValueError(f"set_math: unknown mode {mode!r}: MuZeroModelMLP runs tc3 or tc1")
        code = self.MATH_MODES[mode] if isinstance(mode, str) else int(mode)
        cabi.check(self._lib.lz_model_set_math(self._h, code), "lz_model_set_math")
        self.math = code
        return self

    def eval(self):
        return self

    def to(self, *a, **k):
        return self

    def initial_inference(self, obs: torch.Tensor, return_scalar_value: bool = False) -> MZNetworkOutput:
        """muzero_model_mlp.py:146-178; obs (B, obs_dim)."""
        if not self._loaded:
            raise RuntimeError("MuZeroModelMLP: load_state_dict() has not been called")
        obs = obs.to(self.device, torch.float32).reshape(obs.shape[0], -1).contiguous()
        B = obs.shape[0]
        latent = torch.empty(B, self.latent_state_dim, device=self.device)
        policy = torch.empty(B, self.action_space_size, device=self.device)
        value = torch.empty(B, self.value_support_size, device=self.device)
        scalar = torch.empty(B, device=self.device) if return_scalar_value else None
        with torch.cuda.device(self.device):
            cabi.check(self._lib.lz_model_initial_inference(self._h, B, obs.data_ptr(), latent.data_ptr(), policy.data_ptr(),
                                                            value.data_ptr(), cabi.ptr(scalar), cabi.stream_ptr()),
                       "lz_model_initial_inference")
        out = MZNetworkOutput(value, [0. for _ in range(B)], policy, latent)
        if return_scalar_value:
            out.value_scalar = scalar
        return out

    def recurrent_inference(self, latent_state: torch.Tensor, action: torch.Tensor, return_scalars: bool = False) -> MZNetworkOutput:
        """muzero_model_mlp.py:180-205"""
        if not self._loaded:
            raise RuntimeError("MuZeroModelMLP: load_state_dict() has not been called")
        latent_state = latent_state.to(self.device, torch.float32).contiguous()
        if latent_state.data_ptr() % 16:      # the tensor-core kernel reads latent rows as 16-byte vectors
            latent_state = latent_state.clone()
        action = action.to(self.device).reshape(-1).to(torch.int32).contiguous()
        B = latent_state.shape[0]
        nxt = torch.empty(B, self.latent_state_dim, device=self.device)
        policy = torch.empty(B, self.action_space_size, device=self.device)
        value = torch.empty(B, self.value_support_size, device=self.device)
        reward = torch.empty(B, self.reward_support_size, device=self.device)
        rs = torch.empty(B, device=self.device) if return_scalars else None
        vs = torch.empty(B, device=self.device) if return_scalars else None
        with torch.cuda.device(self.device):
            cabi.check(self._lib.lz_model_recurrent_inference(
                self._h, B, latent_state.data_ptr(), action.data_ptr(), nxt.data_ptr(), reward.data_ptr(), value.data_ptr(),
                policy.data_ptr(), cabi.ptr(rs), cabi.ptr(vs), cabi.stream_ptr()), "lz_model_recurrent_inference")
        out = MZNetworkOutput(value, reward, policy, nxt)
        if return_scalars:
            out.reward_scalar, out.value_scalar = rs, vs
        return out

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                from . import mz_tree
                mz_tree.drop_model_searches(self._serial)
                self._lib.lz_model_destroy(self._h)
        except Exception:
            pass
