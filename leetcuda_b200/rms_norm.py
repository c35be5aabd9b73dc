"""Drop-in mirror of the reference's rms-norm extension (`rms_norm_lib`, kernels/rms-norm/rms_norm.py:10).

Nine ops ``op(x, y, g)`` (kernels/rms-norm/rms_norm.cu:493-771, bound :781-789): ``x``, ``y`` ``[N, K]``
fp32 (``rms_norm_f32``, ``rms_norm_f32x4``) or fp16 (the seven ``rms_norm_f16*`` names), scalar gain
``g``; ``y = x * rsqrt(mean(x^2, dim=1) + 1e-5) * g``, written in place.  The names encode the
reference's vector width and whether its statistics are fp16 or fp32; here every name runs the same
HBM-bound sm_90a kernel (``b200_rms_norm``) with fp32 statistics, which is at least as accurate as each
variant.
"""
from __future__ import annotations

import torch

from . import _capi

_F32 = ["rms_norm_f32", "rms_norm_f32x4"]
_F16 = ["rms_norm_f16_f16", "rms_norm_f16x2_f16", "rms_norm_f16x8_f16", "rms_norm_f16x8_pack_f16",
        "rms_norm_f16x8_f32", "rms_norm_f16x8_pack_f32", "rms_norm_f16_f32"]
OP_NAMES = _F32 + _F16


def rms_norm(x: torch.Tensor, y: torch.Tensor, g: float = 1.0) -> None:
    if x.dtype not in (torch.float32, torch.float16) or y.dtype != x.dtype:
        raise RuntimeError("leetcuda_b200.rms_norm: x and y must both be fp32 or both be fp16")
    if x.dim() != 2 or tuple(y.shape) != tuple(x.shape):
        raise RuntimeError("rms_norm: x and y must be [N, K] of the same shape")
    if not (x.is_cuda and y.is_cuda):
        raise RuntimeError("leetcuda_b200.rms_norm: tensors must be CUDA tensors (no CPU path)")
    if not (x.is_contiguous() and y.is_contiguous()):
        raise RuntimeError("leetcuda_b200.rms_norm: tensors must be contiguous")
    idx = x.device.index
    with torch.cuda.device(idx):
        rc = _capi.lib().b200_rms_norm(x.data_ptr(), y.data_ptr(), float(g), x.size(0), x.size(1),
                                       0 if x.dtype == torch.float32 else 1, _capi.raw_stream(idx))
    _capi.check(rc, "rms_norm")


def _make(name: str, dtype):
    def op(x, y, g: float = 1.0) -> None:
        if x.dtype != dtype or y.dtype != dtype:
            # reference: CHECK_TORCH_TENSOR_DTYPE (rms_norm.cu:421-425)
            raise RuntimeError("values must be torch::kFloat32" if dtype == torch.float32 else "values must be torch::kHalf")
        rms_norm(x, y, g)
    op.__name__ = op.__qualname__ = name
    op.__doc__ = f"{name}(x, y, g) -> None  [sm_90a kernel, fp32 statistics]"
    return op


for _n in _F32:
    globals()[_n] = _make(_n, torch.float32)
for _n in _F16:
    globals()[_n] = _make(_n, torch.float16)

__all__ = OP_NAMES + ["rms_norm", "OP_NAMES"]
