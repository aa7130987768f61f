"""Mirror of lzero/policy/scaling_transform.py:6-13,64-92 (DiscreteSupport, InverseScalarTransform)
for callers that keep their own PyTorch model but want the fused CUDA transform."""
import torch

from . import cabi


class DiscreteSupport(object):
    """scaling_transform.py:6-13"""

    def __init__(self, start: float, stop: float, step: float = 1., device="cuda") -> None:
        assert start < stop
        self.start, self.stop, self.step = float(start), float(stop), float(step)
        self.arange = torch.arange(start, stop, step, dtype=torch.float32).unsqueeze(0).to(device)
        self.size = self.arange.shape[1]
        assert self.size > 0, "DiscreteSupport size must be greater than 0"


class InverseScalarTransform:
    """scaling_transform.py:64-92: softmax(logits) . support -> h^-1, one fused CUDA kernel."""

    def __init__(self, scalar_support: DiscreteSupport, categorical_distribution: bool = True) -> None:
        if not categorical_distribution:
            raise NotImplementedError("only the categorical (support) representation is implemented")
        self.value_support = scalar_support.arange
        self.support = scalar_support
        self._lib = cabi.load()
        cfg = cabi.ModelConfig(4, 84, 84, 1, 1, 64, 16, 16, 16, 32, 32, 32, scalar_support.start,
                               scalar_support.stop, scalar_support.step, downsample=1)
        h = cabi.c_void_p()
        cabi.check(self._lib.lz_model_create(cfg, h), "lz_model_create")
        self._h = h

    def __call__(self, logits: torch.Tensor, epsilon: float = 0.001) -> torch.Tensor:
        assert abs(epsilon - 0.001) < 1e-12, "the kernel fixes epsilon = 0.001 (the reference default)"
        logits = logits.to(torch.float32).contiguous()
        assert logits.is_cuda and logits.shape[1] == self.support.size
        out = torch.empty(logits.shape[0], 1, device=logits.device)
        with torch.cuda.device(logits.device):
            cabi.check(self._lib.lz_inverse_scalar_transform(self._h, logits.shape[0], logits.data_ptr(),
                                                             out.data_ptr(), cabi.stream_ptr()),
                       "lz_inverse_scalar_transform")
        return out

    def __del__(self):
        try:
            self._lib.lz_model_destroy(self._h)
        except Exception:
            pass
