"""Drop-in mirror of the reference's merge_attn_states CUDA extension (SURVEY §8f-3).

Reference: kernels/openai-triton/merge-attn-states/cuda_merge_attn_states.cu:158-177 binds
``merge_attn_states_cuda(output, output_lse, prefix_output, prefix_lse, suffix_output, suffix_lse)``
and cuda_merge_attn_states.py:24-35 wraps it as
``merge_attn_states_cuda(output, prefix_output, prefix_lse, suffix_output, suffix_lse, output_lse=None)``.
Both spellings exist here (``lib.merge_attn_states_cuda`` is the raw binding order) and run the
sm_90a kernel through the C ABI (``b200_merge_attn_states``).

``output`` / ``prefix_output`` / ``suffix_output``: ``[num_tokens, num_heads, head_size]`` fp32, fp16
or bf16; the lse tensors ``[num_heads, num_tokens]`` fp32.  ``output`` (and ``output_lse``) are written
in place.
"""
from __future__ import annotations

from typing import Optional

import torch

from . import _capi

_DTYPES = {torch.float32: 0, torch.float16: 1, torch.bfloat16: 2}


def _bad(name: str, what: str):
    raise RuntimeError(f"merge_attn_states: {name} {what}")


def _raw(output: torch.Tensor, output_lse: Optional[torch.Tensor], prefix_output: torch.Tensor,
         prefix_lse: torch.Tensor, suffix_output: torch.Tensor, suffix_lse: torch.Tensor) -> None:
    # (straight-line checks: at the reference test's sizes the call is launch-bound, every microsecond here shows)
    dt = output.dtype
    code = _DTYPES.get(dt)
    if code is None:
        # reference: TORCH_CHECK(false, "Unsupported data type of O: ", dtype) (cuda_merge_attn_states.cu:107)
        raise RuntimeError(f"Unsupported data type of O: {dt}")
    if output.dim() != 3:
        raise RuntimeError("merge_attn_states: output must be [num_tokens, num_heads, head_size]")
    shape = output.shape
    T, H, D = shape
    pack = 4 if code == 0 else 8
    if D % pack != 0:
        raise RuntimeError(f"headsize must be multiple of pack_size:{pack}")   # :131-132
    if prefix_output.dtype != dt or prefix_output.shape != shape:
        _bad("prefix_output", "must match output in dtype and shape")
    if suffix_output.dtype != dt or suffix_output.shape != shape:
        _bad("suffix_output", "must match output in dtype and shape")
    lshape = (H, T)
    if prefix_lse.dtype != torch.float32 or tuple(prefix_lse.shape) != lshape:
        _bad("prefix_lse", "must be fp32 [num_heads, num_tokens]")
    if suffix_lse.dtype != torch.float32 or tuple(suffix_lse.shape) != lshape:
        _bad("suffix_lse", "must be fp32 [num_heads, num_tokens]")
    lse_ptr = None
    if output_lse is not None:
        if output_lse.dtype != torch.float32 or tuple(output_lse.shape) != lshape:
            _bad("output_lse", "must be fp32 [num_heads, num_tokens]")
        if not (output_lse.is_cuda and output_lse.is_contiguous()):
            _bad("output_lse", "must be a contiguous CUDA tensor")
        lse_ptr = output_lse.data_ptr()
    if not (output.is_cuda and prefix_output.is_cuda and suffix_output.is_cuda and prefix_lse.is_cuda
            and suffix_lse.is_cuda):
        raise RuntimeError("leetcuda_b200.merge_attn_states: tensors must be CUDA tensors (no CPU path)")
    if not (output.is_contiguous() and prefix_output.is_contiguous() and suffix_output.is_contiguous()
            and prefix_lse.is_contiguous() and suffix_lse.is_contiguous()):
        raise RuntimeError("leetcuda_b200.merge_attn_states: tensors must be contiguous")
    idx = output.device.index
    fn = _capi.lib().b200_merge_attn_states
    if torch.cuda.current_device() != idx:
        with torch.cuda.device(idx):
            rc = fn(output.data_ptr(), lse_ptr, prefix_output.data_ptr(), prefix_lse.data_ptr(),
                    suffix_output.data_ptr(), suffix_lse.data_ptr(), T, H, D, code, _capi.raw_stream(idx))
    else:
        rc = fn(output.data_ptr(), lse_ptr, prefix_output.data_ptr(), prefix_lse.data_ptr(),
                suffix_output.data_ptr(), suffix_lse.data_ptr(), T, H, D, code, _capi.raw_stream(idx))
    if rc:
        _capi.check(rc, "merge_attn_states")


def merge_attn_states_cuda(output: torch.Tensor, prefix_output: torch.Tensor, prefix_lse: torch.Tensor,
                           suffix_output: torch.Tensor, suffix_lse: torch.Tensor,
                           output_lse: Optional[torch.Tensor] = None) -> None:
    """cuda_merge_attn_states.py:24-35 (the call the reference's test makes)."""
    _raw(output, output_lse, prefix_output, prefix_lse, suffix_output, suffix_lse)


class lib:  # noqa: N801 — mirrors `lib = load(name="merge_attn_states_cuda", ...)` (cuda_merge_attn_states.py:6)
    """Raw binding order of PYBIND11_MODULE (cuda_merge_attn_states.cu:172-177)."""

    @staticmethod
    def merge_attn_states_cuda(output, output_lse, prefix_output, prefix_lse, suffix_output, suffix_lse) -> None:
        _raw(output, output_lse, prefix_output, prefix_lse, suffix_output, suffix_lse)
