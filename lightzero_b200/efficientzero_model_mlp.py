"""Host-side mirror of ``lzero.model.efficientzero_model_mlp.EfficientZeroModelMLP`` (efficientzero_model_mlp.py:16-300): the
EfficientZero model of the reference's vector-observation configs (cartpole, lunarlander, bipedalwalker, minigrid, pendulum, memory,
bsuite).  Same constructor keywords and defaults, ``initial_inference(obs)`` / ``recurrent_inference(latent_state,
reward_hidden_state, action)`` and ``EZNetworkOutput``; weights from the reference ``state_dict`` (the training-only SSL
``projection`` / ``prediction_head`` entries are ignored).  The dense layers run on the wgmma kernel of csrc/mlp_tc.cu, the
LSTM value-prefix head on ez.cu's; the same object plugs into ``EfficientZeroMCTSCtree.search`` / ``search_with_reuse``
(fused one-graph searches), ``EfficientZeroCollectPolicy`` and the EfficientZero reanalyze.  Inference only (eval mode)."""
from typing import Dict, Optional, Sequence

import torch

from . import cabi
from .efficientzero_model import EZNetworkOutput


class EfficientZeroModelMLP:
    MATH_MODES = {"tc3": 1, "tc1": 2}

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
        if not torch.cuda.is_available():
            raise RuntimeError("lightzero_b200.EfficientZeroModelMLP needs a CUDA device; there is no CPU fallback")
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.observation_shape = int(observation_shape)
        self.action_space_size = int(action_space_size)
        self.latent_state_dim = int(latent_state_dim)
        self.lstm_hidden_size = int(lstm_hidden_size)
        self._lib = cabi.load()
        cfg = cabi.MlpEzConfig(self.observation_shape, self.action_space_size, self.latent_state_dim, self.lstm_hidden_size,
                               reward_head_hidden_channels[0], value_head_hidden_channels[0], policy_head_hidden_channels[0],
                               int(bool(res_connection_in_dynamics)), value_support_range[0], value_support_range[1],
                               value_support_range[2])
        h = cabi.c_void_p()
        with torch.cuda.device(self.device):
            cabi.check(self._lib.lz_model_create_mlp_ez(cfg, h), "lz_model_create_mlp_ez")
        self._h = h
        from .muzero_model import _model_serial
        self._serial = next(_model_serial)      # key of the per-tree lz_search caches (mz_tree)
        self.value_support_size = self.reward_support_size = self._lib.lz_model_support_size(self._h)
        self._loaded = False

    def load_state_dict(self, state_dict: Dict[str, torch.Tensor], strict: bool = True):
        """Takes a reference ``EfficientZeroModelMLP.state_dict()``."""
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
        """'tc3' = wgmma 3xFP16 (fp32-accurate, the default), 'tc1' = wgmma single fp16 pass."""
        if isinstance(mode, str) and mode not in self.MATH_MODES:
            raise ValueError(f"set_math: unknown mode {mode!r}: EfficientZeroModelMLP runs tc3 or tc1")
        code = self.MATH_MODES[mode] if isinstance(mode, str) else int(mode)
        cabi.check(self._lib.lz_model_set_math(self._h, code), "lz_model_set_math")
        self.math = code
        return self

    def eval(self):
        return self

    def to(self, *a, **k):
        return self

    def _check(self):
        if not self._loaded:
            raise RuntimeError("EfficientZeroModelMLP: load_state_dict() has not been called")

    def initial_inference(self, obs: torch.Tensor, return_scalar_value: bool = False) -> EZNetworkOutput:
        """efficientzero_model_mlp.py:150-185; obs (B, obs_dim).  The reward hidden state is zeros (1, B, H)."""
        self._check()
        obs = obs.to(self.device, torch.float32).reshape(obs.shape[0], -1).contiguous()
        B, H = obs.shape[0], self.lstm_hidden_size
        latent = torch.empty(B, self.latent_state_dim, device=self.device)
        policy = torch.empty(B, self.action_space_size, device=self.device)
        value = torch.empty(B, self.value_support_size, device=self.device)
        scalar = torch.empty(B, device=self.device) if return_scalar_value else None
        with torch.cuda.device(self.device):
            cabi.check(self._lib.lz_model_initial_inference(self._h, B, obs.data_ptr(), latent.data_ptr(), policy.data_ptr(),
                                                            value.data_ptr(), cabi.ptr(scalar), cabi.stream_ptr()),
                       "lz_model_initial_inference")
        hidden = (torch.zeros(1, B, H, device=self.device), torch.zeros(1, B, H, device=self.device))
        out = EZNetworkOutput(value, [0. for _ in range(B)], policy, latent, hidden)
        if return_scalar_value:
            out.value_scalar = scalar
        return out

    def recurrent_inference(self, latent_state: torch.Tensor, reward_hidden_state, action: torch.Tensor,
                            return_scalars: bool = False) -> EZNetworkOutput:
        """efficientzero_model_mlp.py:187-300; ``reward_hidden_state`` is the (1, B, H) pair the reference hands to nn.LSTM."""
        self._check()
        latent_state = latent_state.to(self.device, torch.float32).contiguous()
        if latent_state.data_ptr() % 16:      # the kernel reads latent rows as 16-byte vectors
            latent_state = latent_state.clone()
        action = action.to(self.device).reshape(-1).to(torch.int32).contiguous()
        B, H = latent_state.shape[0], self.lstm_hidden_size
        h0 = reward_hidden_state[0].to(self.device, torch.float32).reshape(B, H).contiguous()
        h1 = reward_hidden_state[1].to(self.device, torch.float32).reshape(B, H).contiguous()
        nxt = torch.empty(B, self.latent_state_dim, device=self.device)
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

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                from . import mz_tree
                mz_tree.drop_model_searches(self._serial)     # lz_search handles point at this lz_model: destroy them first
                self._lib.lz_model_destroy(self._h)
        except Exception:
            pass
