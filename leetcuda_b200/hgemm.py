"""Drop-in mirror of the reference's HGEMM extension module (`toy_hgemm` / `hgemm_lib`).

Every name bound in the reference's kernels/hgemm/pybind/hgemm.cc:124-182 exists
here with the same signature, argument meaning and error behaviour:

* 25 three-argument ops            ``op(a, b, c) -> None``
* 13 staged ops                     ``op(a, b, c, stages, swizzle, swizzle_stride) -> None``
* ``init_cublas_handle()`` / ``destroy_cublas_handle()``

``a`` is ``[M,K]`` fp16 row-major, ``c`` is ``[M,N]`` fp16 and is written in
place.  For the NN ops ``b`` is ``[K,N]`` row-major; for the ``*_tn*`` ops ``b``
still has torch shape ``[K,N]`` but its storage is ``[N,K]`` row-major, exactly what
the reference's ``as_col_major`` produces (kernels/hgemm/tools/utils.py:151-156).

All of them run the same sm_90a wgmma/TMA kernel through the C ABI
(``b200_hgemm_f16``); ``stages``/``swizzle``/``swizzle_stride`` are tuning hints of
the reference's own tiling (hgemm.py:198-208) and are accepted and ignored.
Unlike the reference (fp16 accumulation, e.g. mma/basic/hgemm_mma.cu:67-73) the
accumulation is fp32 in the wgmma accumulator registers; see DESIGN.md "Numerics".
"""
from __future__ import annotations

import torch

from . import _capi

__all__ = []  # filled below

# --- op surface (kernels/hgemm/pybind/hgemm.cc:124-182) ----------------------------------
_OPS_3ARG_NN = [
    # naive/hgemm.cu, naive/hgemm_async.cu  (CUDA-core ops; SURVEY §8a row a7)
    "hgemm_naive_f16", "hgemm_sliced_k_f16", "hgemm_t_8x8_sliced_k_f16x4",
    "hgemm_t_8x8_sliced_k_f16x4_pack", "hgemm_t_8x8_sliced_k_f16x4_bcf",
    "hgemm_t_8x8_sliced_k_f16x4_pack_bcf", "hgemm_t_8x8_sliced_k_f16x8_pack_bcf",
    "hgemm_t_8x8_sliced_k_f16x8_pack_bcf_dbuf", "hgemm_t_8x8_sliced_k16_f16x8_pack_dbuf",
    "hgemm_t_8x8_sliced_k16_f16x8_pack_dbuf_async", "hgemm_t_8x8_sliced_k32_f16x8_pack_dbuf",
    "hgemm_t_8x8_sliced_k32_f16x8_pack_dbuf_async", "hgemm_t_16x8_sliced_k32_f16x8_pack_dbuf",
    "hgemm_t_16x8_sliced_k32_f16x8_pack_dbuf_async",
    # wmma/hgemm_wmma.cu (row a4)
    "hgemm_wmma_m16n16k16_naive", "hgemm_wmma_m16n16k16_mma4x2",
    "hgemm_wmma_m16n16k16_mma4x2_warp2x4", "hgemm_wmma_m16n16k16_mma4x2_warp2x4_dbuf_async",
    "hgemm_wmma_m32n8k16_mma2x4_warp2x4_dbuf_async",
    # mma/basic/hgemm_mma.cu (row a2)
    "hgemm_mma_m16n8k16_naive", "hgemm_mma_m16n8k16_mma2x4_warp4x4",
]
_OPS_3ARG_TN = []
_OPS_CUBLAS = ["hgemm_cublas_tensor_op_nn", "hgemm_cublas_tensor_op_tn"]
_OPS_STAGED_NN = [
    "hgemm_wmma_m16n16k16_mma4x2_warp2x4_stages",
    "hgemm_wmma_m16n16k16_mma4x2_warp2x4_stages_dsmem",
    "hgemm_wmma_m16n16k16_mma4x2_warp4x4_stages_dsmem",
    "hgemm_wmma_m16n16k16_mma4x4_warp4x4_stages_dsmem",
    "hgemm_mma_m16n8k16_mma2x4_warp4x4_stages",
    "hgemm_mma_m16n8k16_mma2x4_warp4x4_stages_dsmem",
    "hgemm_mma_m16n8k16_mma2x4_warp4x4x2_stages_dsmem",
    "hgemm_mma_m16n8k16_mma2x4_warp4x4x2_stages_dsmem_x4",
    "hgemm_mma_m16n8k16_mma2x4_warp4x4x2_stages_dsmem_rr",
    "hgemm_mma_m16n8k16_mma2x4_warp4x4x2_stages_dsmem_swizzle",
]
_OPS_STAGED_TN = [
    "hgemm_mma_m16n8k16_mma2x4_warp4x4_stages_dsmem_tn",
    "hgemm_mma_m16n8k16_mma2x4_warp4x4x2_stages_dsmem_tn_swizzle_x4",
    "hgemm_mma_stages_block_swizzle_tn_cute",
]
OP_NAMES = _OPS_3ARG_NN + _OPS_3ARG_TN + _OPS_CUBLAS + _OPS_STAGED_NN + _OPS_STAGED_TN


def _check_half(t: torch.Tensor) -> None:
    # reference: CHECK_TORCH_TENSOR_DTYPE (mma/basic/hgemm_mma.cu:295-299)
    if t.dtype != torch.float16:
        raise RuntimeError("values must be torch::kHalf")


def _check_shape(t: torch.Tensor, s0: int, s1: int) -> None:
    # reference: CHECK_TORCH_TENSOR_SHAPE (mma/basic/hgemm_mma.cu:301-304)
    if t.dim() != 2 or t.size(0) != s0 or t.size(1) != s1:
        raise RuntimeError("Tensor size mismatch!")


import os

# LEETCUDA_B200_HGEMM_ACC=f16: every mirror op accumulates in fp16 like the reference (parity mode)
_DEFAULT_ACC = os.environ.get("LEETCUDA_B200_HGEMM_ACC", "f32").lower()


def hgemm(a: torch.Tensor, b: torch.Tensor, c: torch.Tensor, *, tn: bool = False,
          acc: str = "") -> None:
    """``c[M,N] = a[M,K] @ B`` on the current CUDA stream of ``a``'s device.

    ``tn=False``: ``b`` is ``[K,N]`` row-major.  ``tn=True``: ``b`` has shape ``[K,N]``
    but holds ``[N,K]`` row-major storage (the reference's TN convention).
    ``acc``: ``"f32"`` (default, fp32 accumulators) or ``"f16"`` (the reference's fp16
    accumulation, for bit-level comparison with its kernels).
    """
    _check_half(a)
    _check_half(b)
    _check_half(c)
    M, K = a.size(0), a.size(1)
    N = b.size(1)
    _check_shape(a, M, K)
    _check_shape(b, K, N)
    _check_shape(c, M, N)
    if not (a.is_cuda and b.is_cuda and c.is_cuda):
        raise RuntimeError("leetcuda_b200.hgemm: tensors must be CUDA tensors (no CPU path)")
    if not (a.is_contiguous() and b.is_contiguous() and c.is_contiguous()):
        raise RuntimeError("leetcuda_b200.hgemm: tensors must be contiguous")
    lib = _capi.lib()
    fn = lib.b200_hgemm_f16_acc16 if (acc or _DEFAULT_ACC) == "f16" else lib.b200_hgemm_f16
    idx = a.device.index
    layout = _capi.B_ROW_MAJOR_NK if tn else _capi.B_ROW_MAJOR_KN
    if torch.cuda.current_device() != idx:   # launch on the tensors' device, as the op contract requires
        with torch.cuda.device(idx):
            rc = fn(a.data_ptr(), b.data_ptr(), c.data_ptr(), M, N, K, layout, _capi.raw_stream(idx))
    else:
        rc = fn(a.data_ptr(), b.data_ptr(), c.data_ptr(), M, N, K, layout, _capi.raw_stream(idx))
    _capi.check(rc, "hgemm")


def hgemm_ex(a, b, c, *, tn=False, cta_group=0, group_m=0, max_ctas=0, b_lbo=0, b_sbo=0,
             b_kstep=0) -> None:
    """Same as :func:`hgemm` with the tuning/debug knobs of ``b200_hgemm_f16_ex``."""
    _check_half(a); _check_half(b); _check_half(c)
    M, K = a.size(0), a.size(1)
    N = b.size(1)
    _check_shape(b, K, N)
    _check_shape(c, M, N)
    rc = _capi.lib().b200_hgemm_f16_ex(
        a.data_ptr(), b.data_ptr(), c.data_ptr(), M, N, K,
        _capi.B_ROW_MAJOR_NK if tn else _capi.B_ROW_MAJOR_KN,
        cta_group, group_m, max_ctas, b_lbo, b_sbo, b_kstep,
        torch.cuda.current_stream(a.device).cuda_stream)
    _capi.check(rc, "hgemm_ex")


def hgemm_host(a: torch.Tensor, b: torch.Tensor, c: torch.Tensor, *, tn: bool = False) -> None:
    """Host-buffer entry point (``b200_hgemm_f16_host``): ``a``, ``b``, ``c`` are CPU tensors
    (pinned for full PCIe rate).  Copies in, multiplies on the current device and copies out,
    pipelined over row panels; returns when ``c`` is complete.  Used for end-to-end timing."""
    _check_half(a); _check_half(b); _check_half(c)
    M, K = a.size(0), a.size(1)
    N = b.size(1)
    _check_shape(b, K, N)
    _check_shape(c, M, N)
    if a.is_cuda or b.is_cuda or c.is_cuda:
        raise RuntimeError("leetcuda_b200.hgemm_host: tensors must be host tensors")
    idx = torch.cuda.current_device()
    rc = _capi.lib().b200_hgemm_f16_host(a.data_ptr(), b.data_ptr(), c.data_ptr(), M, N, K,
                                         _capi.B_ROW_MAJOR_NK if tn else _capi.B_ROW_MAJOR_KN,
                                         _capi.raw_stream(idx))
    _capi.check(rc, "hgemm_host")


def _make_3arg(name: str, tn: bool):
    def op(a: torch.Tensor, b: torch.Tensor, c: torch.Tensor) -> None:
        hgemm(a, b, c, tn=tn)
    op.__name__ = op.__qualname__ = name
    op.__doc__ = f"{name}(a, b, c) -> None  [{'TN' if tn else 'NN'}; sm_90a wgmma kernel]"
    return op


def _make_staged(name: str, tn: bool):
    def op(a: torch.Tensor, b: torch.Tensor, c: torch.Tensor, stages: int = 2,
           swizzle: bool = False, swizzle_stride: int = 1) -> None:
        hgemm(a, b, c, tn=tn)
    op.__name__ = op.__qualname__ = name
    op.__doc__ = (f"{name}(a, b, c, stages, swizzle, swizzle_stride) -> None  "
                  f"[{'TN' if tn else 'NN'}; hints ignored; sm_90a wgmma kernel]")
    return op


for _n in _OPS_3ARG_NN:
    globals()[_n] = _make_3arg(_n, False)
for _n in _OPS_3ARG_TN:
    globals()[_n] = _make_3arg(_n, True)
for _n in _OPS_STAGED_NN:
    globals()[_n] = _make_staged(_n, False)
for _n in _OPS_STAGED_TN:
    globals()[_n] = _make_staged(_n, True)


def hgemm_cublas_tensor_op_nn(a: torch.Tensor, b: torch.Tensor, c: torch.Tensor) -> None:
    """Vendor row (reference: cublas/hgemm_cublas.cu:41-54, cublasGemmEx): stays a cuBLAS
    call (through torch.matmul) so the scripts' "cublas" rows remain the vendor baseline
    rather than silently becoming this library's kernel."""
    _check_half(a); _check_half(b); _check_half(c)
    _check_shape(b, a.size(1), b.size(1)); _check_shape(c, a.size(0), b.size(1))
    torch.matmul(a, b, out=c)


def hgemm_cublas_tensor_op_tn(a: torch.Tensor, b: torch.Tensor, c: torch.Tensor) -> None:
    """Vendor row, TN (reference: cublas/hgemm_cublas.cu:56-68); b holds [N,K] storage."""
    _check_half(a); _check_half(b); _check_half(c)
    K, N = b.size(0), b.size(1)
    _check_shape(c, a.size(0), N)
    torch.matmul(a, b.view(N, K).t(), out=c)


def init_cublas_handle() -> None:
    """reference: cublas/hgemm_cublas.cu:15-25.  No handle is needed here; kept for the
    scripts that bracket the cublas rows with init/destroy (hgemm.py:243-244,321-322)."""
    _capi.lib()


def destroy_cublas_handle() -> None:
    """reference: cublas/hgemm_cublas.cu:27-38 (no-op here)."""


__all__ = OP_NAMES + ["init_cublas_handle", "destroy_cublas_handle", "hgemm", "hgemm_ex", "hgemm_host",
                      "OP_NAMES"]
