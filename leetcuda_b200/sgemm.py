"""Drop-in mirror of the reference's SGEMM extension module (`sgemm_lib`), SURVEY §8f-2.

Every name bound in the reference's kernels/sgemm/sgemm.cu:743-765 exists here with the same
signature, argument meaning and error behaviour.  ``a`` is ``[M,K]``, ``b`` is ``[K,N]``, ``c`` is
``[M,N]``, all fp32 row-major; ``c`` is written in place.

* the two TF32 tensor-core ops
  ``sgemm_wmma_m16n16k8_mma4x2_warp2x4_stages{,_dsmem}(a, b, c, stages, swizzle, swizzle_stride)``
  (sgemm_wmma_tf32_stage.cu:573-742) run the sm_90a wgmma ``.tf32`` kernel through the
  C ABI (``b200_sgemm_tf32``).  Like the reference they first round ``a`` and ``b`` to TF32 **in
  place** (sgemm_wmma_tf32_stage.cu:44-60, 586-592); the hints are accepted and ignored.
* ``sgemm_cublas`` / ``sgemm_cublas_tf32`` (sgemm_cublas.cu:17-43) stay vendor calls: they are the
  vendor rows of the reference's table and say so in their docstrings.
* the 13 CUDA-core fp32 ops (sgemm.cu:743-760, sgemm_async.cu) compute a full-precision fp32 product (FFMA
  accumulation, ~2e-6 relative at K = 1024).  No tensor-core path reproduces that: a TF32 product is at 1e-3,
  and the 3xTF32 split offered here as ``sgemm_3xtf32`` (``b200_sgemm_3xtf32``: each operand = two exact TF32
  numbers, three partial products in ONE wgmma ``.tf32`` GEMM over K' = 3K) removes the operand rounding
  but keeps the tensor core's truncating accumulation — measured 5e-5 relative at K = 1024..4096
  (tests/test_sgemm_gpu.py), 20x better than TF32 and 20x worse than FFMA.  So by default these 13 names are
  VENDOR ROWS (cuBLAS fp32 through torch.matmul, said so in every docstring) and keep the reference's
  accuracy; ``LEETCUDA_B200_SGEMM_FP32=3xtf32`` routes them through the 3xTF32 kernel instead (about 4x the
  vendor fp32 rate at 8192^3).
"""
from __future__ import annotations

import torch

from . import _capi

_OPS_FP32_CUDA_CORE = [
    "sgemm_naive_f32", "sgemm_sliced_k_f32", "sgemm_t_8x8_sliced_k_f32x4",
    "sgemm_t_8x8_sliced_k_f32x4_bcf", "sgemm_t_8x8_sliced_k_f32x4_bcf_offset",
    "sgemm_t_8x8_sliced_k_f32x4_bcf_dbuf", "sgemm_t_8x8_sliced_k_f32x4_bcf_dbuf_offset",
    "sgemm_t_8x4_sliced_k16_f32x4_bcf_dbuf", "sgemm_t_8x4_sliced_k16_f32x4_bcf_dbuf_async",
    "sgemm_t_8x8_sliced_k16_f32x4_bcf_dbuf", "sgemm_t_8x8_sliced_k16_f32x4_bcf_dbuf_async",
    "sgemm_t_8x16_sliced_k16_f32x4_bcf_dbuf", "sgemm_t_8x16_sliced_k16_f32x4_bcf_dbuf_async",
]
_OPS_CUBLAS = ["sgemm_cublas", "sgemm_cublas_tf32"]
_OPS_TF32_STAGED = ["sgemm_wmma_m16n16k8_mma4x2_warp2x4_stages",
                    "sgemm_wmma_m16n16k8_mma4x2_warp2x4_stages_dsmem"]
OP_NAMES = _OPS_FP32_CUDA_CORE + _OPS_CUBLAS + _OPS_TF32_STAGED
__all__ = OP_NAMES + ["sgemm_tf32", "sgemm_3xtf32", "tf32_round_", "OP_NAMES"]


def _check_f32(t: torch.Tensor) -> None:
    # reference: CHECK_TORCH_TENSOR_DTYPE(T, torch::kFloat32) (sgemm_wmma_tf32_stage.cu:576-578)
    if t.dtype != torch.float32:
        raise RuntimeError("values must be torch::kFloat32")


def _check_shape(t: torch.Tensor, s0: int, s1: int) -> None:
    # reference: CHECK_TORCH_TENSOR_SHAPE (sgemm_wmma_tf32_stage.cu:582-584)
    if t.dim() != 2 or t.size(0) != s0 or t.size(1) != s1:
        raise RuntimeError("Tensor size mismatch!")


def _check_all(a, b, c):
    _check_f32(a); _check_f32(b); _check_f32(c)
    M, K = a.size(0), a.size(1)
    N = b.size(1)
    _check_shape(a, M, K)
    _check_shape(b, K, N)
    _check_shape(c, M, N)
    return M, N, K


def _check_device(*ts):
    if not all(t.is_cuda for t in ts):
        raise RuntimeError("leetcuda_b200.sgemm: tensors must be CUDA tensors (no CPU path)")
    if not all(t.is_contiguous() for t in ts):
        raise RuntimeError("leetcuda_b200.sgemm: tensors must be contiguous")


def sgemm_tf32(a: torch.Tensor, b: torch.Tensor, c: torch.Tensor, *, tn: bool = False,
               round_inputs: bool = True) -> None:
    """``c[M,N] = tf32(a)[M,K] @ tf32(B)`` with fp32 accumulation, on the current stream of ``a``'s device.

    ``round_inputs=True`` (the reference's behaviour) rewrites ``a`` and ``b`` with their TF32
    roundings before the product; ``False`` leaves them untouched (the tensor core then truncates).
    ``tn=True``: ``b`` has shape ``[K,N]`` but ``[N,K]`` row-major storage (no reference counterpart).
    """
    M, N, K = _check_all(a, b, c)
    _check_device(a, b, c)
    idx = a.device.index
    layout = _capi.B_ROW_MAJOR_NK if tn else _capi.B_ROW_MAJOR_KN
    fn = _capi.lib().b200_sgemm_tf32
    if torch.cuda.current_device() != idx:
        with torch.cuda.device(idx):
            rc = fn(a.data_ptr(), b.data_ptr(), c.data_ptr(), M, N, K, layout, int(round_inputs),
                    _capi.raw_stream(idx))
    else:
        rc = fn(a.data_ptr(), b.data_ptr(), c.data_ptr(), M, N, K, layout, int(round_inputs),
                _capi.raw_stream(idx))
    _capi.check(rc, "sgemm_tf32")


def tf32_round_(x: torch.Tensor) -> torch.Tensor:
    """In-place TF32 rounding (``b200_tf32_round_inplace``), the reference's f32x4_tf32x4_kernel."""
    _check_f32(x)
    _check_device(x)
    rc = _capi.lib().b200_tf32_round_inplace(x.data_ptr(), x.numel(),
                                             torch.cuda.current_stream(x.device).cuda_stream)
    _capi.check(rc, "tf32_round")
    return x


def _make_tf32_staged(name: str):
    def op(a: torch.Tensor, b: torch.Tensor, c: torch.Tensor, stages: int = 2,
           swizzle: bool = False, swizzle_stride: int = 1) -> None:
        sgemm_tf32(a, b, c, round_inputs=True)
    op.__name__ = op.__qualname__ = name
    op.__doc__ = (f"{name}(a, b, c, stages, swizzle, swizzle_stride) -> None  "
                  "[TF32 tensor cores, inputs rounded in place; hints ignored; sm_90a wgmma kernel]")
    return op


def _vendor_fp32(a, b, c, allow_tf32: bool) -> None:
    _check_all(a, b, c)
    prev = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = allow_tf32
    try:
        torch.matmul(a, b, out=c)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = prev


def sgemm_3xtf32(a: torch.Tensor, b: torch.Tensor, c: torch.Tensor) -> None:
    """``c = a @ b`` on the TF32 tensor cores through the 3xTF32 split (``b200_sgemm_3xtf32``): exact operands, the
    tensor core's accumulation — about 5e-5 relative at K = 1024..4096, between TF32 (1e-3) and FFMA fp32 (2e-6)."""
    M, N, K = _check_all(a, b, c)
    _check_device(a, b, c)
    idx = a.device.index
    with torch.cuda.device(idx):
        rc = _capi.lib().b200_sgemm_3xtf32(a.data_ptr(), b.data_ptr(), c.data_ptr(), M, N, K, _capi.raw_stream(idx))
    _capi.check(rc, "sgemm_3xtf32")


def _fp32_mode() -> str:
    import os
    return os.environ.get("LEETCUDA_B200_SGEMM_FP32", "vendor")


def _make_fp32(name: str):
    def op(a: torch.Tensor, b: torch.Tensor, c: torch.Tensor) -> None:
        if _fp32_mode() == "3xtf32":
            sgemm_3xtf32(a, b, c)
        else:
            _vendor_fp32(a, b, c, False)
    op.__name__ = op.__qualname__ = name
    op.__doc__ = (f"{name}(a, b, c) -> None  [VENDOR ROW by default: cuBLAS fp32 through torch.matmul, not a kernel of this "
                  "library (full fp32 accuracy like the reference's FFMA kernel); LEETCUDA_B200_SGEMM_FP32=3xtf32 selects "
                  "the 3xTF32 tensor-core kernel]")
    return op


for _n in _OPS_TF32_STAGED:
    globals()[_n] = _make_tf32_staged(_n)
for _n in _OPS_FP32_CUDA_CORE:
    globals()[_n] = _make_fp32(_n)


def sgemm_cublas(a: torch.Tensor, b: torch.Tensor, c: torch.Tensor) -> None:
    """VENDOR ROW — cuBLAS fp32 through torch.matmul, not a kernel of this library (reference: sgemm_cublas.cu:17-29,
    CUBLAS_DEFAULT_MATH / COMPUTE_32F; kept a vendor call so the scripts' "cublas" rows keep their meaning)."""
    _vendor_fp32(a, b, c, False)


def sgemm_cublas_tf32(a: torch.Tensor, b: torch.Tensor, c: torch.Tensor) -> None:
    """VENDOR ROW — cuBLAS TF32 through torch.matmul, not a kernel of this library (reference: sgemm_cublas.cu:31-43,
    CUBLAS_TF32_TENSOR_OP_MATH)."""
    _vendor_fp32(a, b, c, True)
