"""What the CUDA model wrappers (``MuZeroModel``, ``EfficientZeroModel``, ``MuZeroModelMLP``, ``EfficientZeroModelMLP`` and
the two Stochastic MuZero models) share: one ``lz_model`` handle and its lifecycle, the weights from a reference
``state_dict``, the math mode, and the inference bodies.  The model family is the class-level ``value_prefix`` flag: the
EfficientZero models carry the LSTM value-prefix head, their ``recurrent_inference`` takes and returns the reward hidden state
and their searches run on value-prefix trees; the Stochastic MuZero models (``StochasticLzModel``) run on stochastic trees."""
import itertools
from dataclasses import dataclass
from typing import Dict, Tuple

import torch

from . import cabi, mz_tree
from .scaling_transform import check_support

_model_serial = itertools.count(1)      # never reused (unlike id()): keys of the per-tree lz_search caches in mz_tree


@dataclass
class MZNetworkOutput:
    """lzero/model/common.py:131-141"""
    value: torch.Tensor
    reward: torch.Tensor
    policy_logits: torch.Tensor
    latent_state: torch.Tensor


@dataclass
class EZNetworkOutput:
    """lzero/model/common.py:119-128"""
    value: torch.Tensor
    value_prefix: torch.Tensor
    policy_logits: torch.Tensor
    latent_state: torch.Tensor
    reward_hidden_state: Tuple[torch.Tensor, torch.Tensor]


class LzModel:
    """Base of the model wrappers.  A subclass validates its keywords, calls ``_create`` and sets ``_latent``, the shape of
    one root's latent: (C, H, W) for the conv models, (latent_state_dim,) for the MLP models."""
    value_prefix = False        # the EfficientZero family
    _align_latents = False      # the MLP kernels read latent rows as 16-byte vectors
    MATH_MODES = {"tc3": 1, "tc1": 2}

    def _create(self, device, create: str, cfg, support_range):
        check_support(support_range)
        if not torch.cuda.is_available():
            raise RuntimeError(f"lightzero_b200.{type(self).__name__} needs a CUDA device; there is no CPU fallback")
        self.device = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        self._lib = cabi.load()
        h = cabi.c_void_p()
        with torch.cuda.device(self.device):
            cabi.check(getattr(self._lib, create)(cfg, h), create)
        self._h = h
        self._serial = next(_model_serial)
        self.value_support_size = self.reward_support_size = self._lib.lz_model_support_size(self._h)
        self._loaded = False

    # ---- weights -------------------------------------------------------------------------------
    def load_state_dict(self, state_dict: Dict[str, torch.Tensor], strict: bool = True):
        """Takes the reference model's ``state_dict()`` (SURVEY.md App. B.4 key layout)."""
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
        """'tc3' = wgmma 3xFP16 (fp32-accurate, the default), 'tc1' = wgmma single fp16 pass.  A MuZeroModelMLP on the fp32
        kernels has no math mode (LzError)."""
        if isinstance(mode, str) and mode not in self.MATH_MODES:
            raise ValueError(f"set_math: unknown mode {mode!r}: {type(self).__name__} runs tc3 or tc1")
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
            raise RuntimeError(f"{type(self).__name__}: load_state_dict() has not been called")

    def initial_inference(self, obs: torch.Tensor, return_scalar_value: bool = False):
        """muzero_model.py:210-240 / efficientzero_model.py:203-238.  ``reward`` / ``value_prefix`` is the python list of zeros
        the reference returns; an EfficientZero model's reward hidden state is zeros (1, B, lstm_hidden_size)."""
        self._check()
        d = self.device
        obs = obs.to(d, torch.float32).reshape(obs.shape[0], -1).contiguous()
        B = obs.shape[0]
        latent = torch.empty((B,) + self._latent, device=d)
        policy = torch.empty(B, self.action_space_size, device=d)
        value = torch.empty(B, self.value_support_size, device=d)
        scalar = torch.empty(B, device=d) if return_scalar_value else None
        with torch.cuda.device(d):
            cabi.check(self._lib.lz_model_initial_inference(self._h, B, obs.data_ptr(), latent.data_ptr(), policy.data_ptr(),
                                                            value.data_ptr(), cabi.ptr(scalar), cabi.stream_ptr()),
                       "lz_model_initial_inference")
        if self.value_prefix:
            H = self.lstm_hidden_size
            hidden = (torch.zeros(1, B, H, device=d), torch.zeros(1, B, H, device=d))
            out = EZNetworkOutput(value, [0. for _ in range(B)], policy, latent, hidden)
        else:
            out = MZNetworkOutput(value, [0. for _ in range(B)], policy, latent)
        if return_scalar_value:
            out.value_scalar = scalar
        return out

    def recurrent_inference(self, latent_state: torch.Tensor, action: torch.Tensor, return_scalars: bool = False):
        """muzero_model.py:242-272; ``action`` is (B,) or (B,1) integer."""
        return self._recurrent(latent_state, None, action, return_scalars)

    def _recurrent(self, latent_state, reward_hidden_state, action, return_scalars):
        """recurrent_inference of either family; ``reward_hidden_state`` is the EfficientZero (1, B, H) pair the reference
        hands to nn.LSTM."""
        self._check()
        d = self.device
        latent_state = latent_state.to(d, torch.float32).contiguous()
        if self._align_latents and latent_state.data_ptr() % 16:
            latent_state = latent_state.clone()
        action = action.to(d).reshape(-1).to(torch.int32).contiguous()
        B = latent_state.shape[0]
        nxt = torch.empty((B,) + self._latent, device=d)
        policy = torch.empty(B, self.action_space_size, device=d)
        value = torch.empty(B, self.value_support_size, device=d)
        reward = torch.empty(B, self.reward_support_size, device=d)      # the value prefix for EfficientZero
        rs = torch.empty(B, device=d) if return_scalars else None
        vs = torch.empty(B, device=d) if return_scalars else None
        with torch.cuda.device(d):
            if not self.value_prefix:
                cabi.check(self._lib.lz_model_recurrent_inference(
                    self._h, B, latent_state.data_ptr(), action.data_ptr(), nxt.data_ptr(), reward.data_ptr(), value.data_ptr(),
                    policy.data_ptr(), cabi.ptr(rs), cabi.ptr(vs), cabi.stream_ptr()), "lz_model_recurrent_inference")
                out = MZNetworkOutput(value, reward, policy, nxt)
                if return_scalars:
                    out.reward_scalar, out.value_scalar = rs, vs
                return out
            H = self.lstm_hidden_size
            h0 = reward_hidden_state[0].to(d, torch.float32).reshape(B, H).contiguous()
            h1 = reward_hidden_state[1].to(d, torch.float32).reshape(B, H).contiguous()
            n0, n1 = torch.empty(1, B, H, device=d), torch.empty(1, B, H, device=d)
            cabi.check(self._lib.lz_model_recurrent_inference_ez(
                self._h, B, latent_state.data_ptr(), h0.data_ptr(), h1.data_ptr(), action.data_ptr(), nxt.data_ptr(),
                n0.data_ptr(), n1.data_ptr(), reward.data_ptr(), value.data_ptr(), policy.data_ptr(), cabi.ptr(rs),
                cabi.ptr(vs), cabi.stream_ptr()), "lz_model_recurrent_inference_ez")
        out = EZNetworkOutput(value, reward, policy, nxt, (n0, n1))
        if return_scalars:
            out.value_prefix_scalar, out.value_scalar = rs, vs
        return out

    def __del__(self):
        try:
            if getattr(self, "_h", None):
                mz_tree.drop_model_searches(self._serial)     # lz_search handles point at this lz_model: destroy them first
                self._lib.lz_model_destroy(self._h)
        except Exception:
            pass


class StochasticLzModel(LzModel):
    """Base of the Stochastic MuZero wrappers (``StochasticMuZeroModelMLP``, ``StochasticMuZeroModel``): a subclass sets
    ``chance_space_size``.  Their searches run on stochastic trees, and ``recurrent_inference`` takes the reference's
    ``afterstate`` flag."""
    chance_space_size = 0

    def recurrent_inference(self, state: torch.Tensor, option: torch.Tensor, afterstate: bool = False,
                            return_scalars: bool = False) -> MZNetworkOutput:
        """stochastic_muzero_model.py:233-273.  ``afterstate=False``: ``state`` is a latent and ``option`` an action; returns
        the afterstate and its chance logits [B, chance_space_size].  ``afterstate=True``: ``state`` is an afterstate and
        ``option`` a chance outcome; returns the next latent and its policy logits [B, action_space_size]."""
        self._check()
        d = self.device
        state = state.to(d, torch.float32).contiguous()
        if self._align_latents and state.data_ptr() % 16:
            state = state.clone()
        option = option.to(d).reshape(-1).to(torch.int32).contiguous()
        B = state.shape[0]
        nxt = torch.empty((B,) + self._latent, device=d)
        policy = torch.empty(B, self.action_space_size if afterstate else self.chance_space_size, device=d)
        value = torch.empty(B, self.value_support_size, device=d)
        reward = torch.empty(B, self.reward_support_size, device=d)
        rs = torch.empty(B, device=d) if return_scalars else None
        vs = torch.empty(B, device=d) if return_scalars else None
        with torch.cuda.device(d):
            cabi.check(self._lib.lz_model_recurrent_inference_stochastic(
                self._h, int(bool(afterstate)), B, state.data_ptr(), option.data_ptr(), None, 0, nxt.data_ptr(),
                reward.data_ptr(), value.data_ptr(), policy.data_ptr(), cabi.ptr(rs), cabi.ptr(vs), cabi.stream_ptr()),
                "lz_model_recurrent_inference_stochastic")
        out = MZNetworkOutput(value, reward, policy, nxt)
        if return_scalars:
            out.reward_scalar, out.value_scalar = rs, vs
        return out
