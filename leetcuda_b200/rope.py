"""Drop-in mirror of the reference's rope extension (`lib = load(name="rope", ...)`, kernels/rope/rope.py:10).

``rope_f32(x, out)``, ``rope_f32_v2(x, out)``, ``rope_f32x4_pack(x, out)`` (kernels/rope/rope.cu:88-125):
``x``, ``out`` fp32 ``[seq_len, hidden]``; the three names differ only in the reference's thread indexing,
here they run the same HBM-bound sm_90a kernel through ``b200_rope_f32``.  ``out`` is written in place.
"""
from __future__ import annotations

import torch

from . import _capi


def _rope(x: torch.Tensor, out: torch.Tensor) -> None:
    if x.dtype != torch.float32 or out.dtype != torch.float32:
        raise RuntimeError("values must be torch::kFloat32")          # rope.cu:89-90
    if x.dim() != 2 or tuple(out.shape) != tuple(x.shape):
        raise RuntimeError("rope: x and out must be [seq_len, hidden] of the same shape")
    if not (x.is_cuda and out.is_cuda):
        raise RuntimeError("leetcuda_b200.rope: tensors must be CUDA tensors (no CPU path)")
    if not (x.is_contiguous() and out.is_contiguous()):
        raise RuntimeError("leetcuda_b200.rope: tensors must be contiguous")
    idx = x.device.index
    with torch.cuda.device(idx):
        rc = _capi.lib().b200_rope_f32(x.data_ptr(), out.data_ptr(), x.size(0), x.size(1), _capi.raw_stream(idx))
    _capi.check(rc, "rope_f32")


def rope_f32(x, out) -> None:
    """reference: rope.cu:88-99."""
    _rope(x, out)


def rope_f32_v2(x, out) -> None:
    """reference: rope.cu:101-112."""
    _rope(x, out)


def rope_f32x4_pack(x, out) -> None:
    """reference: rope.cu:114-125."""
    _rope(x, out)


OP_NAMES = ["rope_f32", "rope_f32_v2", "rope_f32x4_pack"]
__all__ = OP_NAMES + ["OP_NAMES"]
