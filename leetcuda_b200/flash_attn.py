"""Drop-in mirror of the reference's FlashAttention extension module (`flash_attn_lib`).

Every name bound in the reference's kernels/flash-attn/pybind/flash_attn.cc:168-224
exists here with the same signature and error behaviour:

* 28 ops  ``op(Q, K, V, O, stages) -> None``  (6 basic, 4 acc_f32, 15 swizzle, 3 "others")
* ``flash_attn_cute(Q, K, V, O) -> None``

Q, K, O are fp16 contiguous ``[B,H,N,D]``; V is ``[B,H,N,D]`` except for the three
``*_swizzle_qkv`` ops of the share-kv / share-qkv / tiling-qk families, which take V
pre-transposed ``[B,H,D,N]`` (flash_attn_mma.py:441-442,716,807,898).  O is written
in place.  Non-causal, scale = 1/sqrt(D) (flash_attn_mma_split_q.cu:79).

All of them run the same fused sm_90a kernel through ``b200_fmha_fwd_f16``;
``stages`` is a hint of the reference's cp.async pipeline and is ignored.  The
reference's family differences (which of Q/K/V share smem, fp16 vs fp32 MMA
accumulators) are implementation details of its mma.sync kernels: here S and O
always accumulate in fp32 in registers, which is at least as accurate as every variant.
"""
from __future__ import annotations

import math

import torch

from . import _capi

_BASIC = [
    "flash_attn_mma_stages_split_kv", "flash_attn_mma_stages_split_q",
    "flash_attn_mma_stages_split_q_shared_kv", "flash_attn_mma_stages_split_q_shared_qkv",
    "flash_attn_mma_stages_split_q_tiling_qk", "flash_attn_mma_stages_split_q_tiling_qkv",
]
_ACC_F32 = [
    "flash_attn_mma_stages_split_q_shared_kv_acc_f32",
    "flash_attn_mma_stages_split_q_shared_qkv_acc_f32",
    "flash_attn_mma_stages_split_q_tiling_qk_acc_f32",
    "flash_attn_mma_stages_split_q_tiling_qkv_acc_f32",
]
_SWIZZLE = [
    "flash_attn_mma_stages_split_q_shared_kv_swizzle_q",
    "flash_attn_mma_stages_split_q_shared_kv_swizzle_qk",
    "flash_attn_mma_stages_split_q_shared_kv_swizzle_qkv",
    "flash_attn_mma_stages_split_q_shared_qkv_swizzle_q",
    "flash_attn_mma_stages_split_q_shared_qkv_swizzle_qk",
    "flash_attn_mma_stages_split_q_shared_qkv_swizzle_qkv",
    "flash_attn_mma_stages_split_q_tiling_qk_swizzle_q",
    "flash_attn_mma_stages_split_q_tiling_qk_swizzle_qk",
    "flash_attn_mma_stages_split_q_tiling_qk_swizzle_qkv",
    "flash_attn_mma_stages_split_q_tiling_qkv_swizzle_q",
    "flash_attn_mma_stages_split_q_tiling_qkv_swizzle_qk",
    "flash_attn_mma_stages_split_q_tiling_qkv_swizzle_qkv",
    "flash_attn_mma_stages_split_q_tiling_qkv_acc_f32_swizzle_q",
    "flash_attn_mma_stages_split_q_tiling_qkv_acc_f32_swizzle_qk",
    "flash_attn_mma_stages_split_q_tiling_qkv_acc_f32_swizzle_qkv",
]
_OTHERS = [  # only under -DBUILD_FLASH_ATTN_MMA_OTHERS in the reference (flash_attn.cc:217-223)
    "flash_attn_mma_stages_split_q_shared_qkv_Os2g",
    "flash_attn_mma_stages_split_q_shared_kv_acc_f32_rr",
    "flash_attn_mma_stages_split_q_shared_qkv_acc_f32_rr",
]
# ops whose V argument is [B,H,D,N]
V_TRANSPOSED_OPS = {
    "flash_attn_mma_stages_split_q_shared_kv_swizzle_qkv",
    "flash_attn_mma_stages_split_q_shared_qkv_swizzle_qkv",
    "flash_attn_mma_stages_split_q_tiling_qk_swizzle_qkv",
}
OP_NAMES = _BASIC + _ACC_F32 + _SWIZZLE + _OTHERS


def _shapes(Q, K, V, O, v_transposed, same_length, grouped=False, dtype=torch.float16, fp8=False):
    """(B, H, Nq, Nk, D, Hkv) of q, o [B,H,Nq,D], k [B,Hkv,Nk,D], v [B,Hkv,Nk,D] or [B,Hkv,D,Nk]; Nk = Nq if
    same_length; Hkv = H unless grouped, where any Hkv dividing H is accepted.  fp8: the dtypes were checked by
    _fp8_kv."""
    if not fp8:
        _check_dtype(Q, K, V, O, dtype)
    if Q.dim() != 4 or K.dim() != 4:
        raise RuntimeError("Tensor size mismatch!")
    B, H, Nq, D = Q.shape
    Nk = Nq if same_length else K.shape[2]
    Hkv = K.shape[1] if grouped and K.shape[1] > 0 and H % K.shape[1] == 0 else H
    if tuple(K.shape) != (B, Hkv, Nk, D) or tuple(O.shape) != (B, H, Nq, D):
        raise RuntimeError("Tensor size mismatch!")
    want_v = (B, Hkv, D, Nk) if v_transposed else (B, Hkv, Nk, D)
    if tuple(V.shape) != want_v:
        raise RuntimeError("Tensor size mismatch!")
    return B, H, Nq, Nk, D, Hkv


def _check_dtype(Q, K, V, O, dtype):
    for t in (Q, K, V, O):
        if t.dtype != dtype:
            raise RuntimeError("values must be torch::kHalf" if dtype == torch.float16 else "values must be torch::kBFloat16")


def _element_type(Q, K, V, O):
    """torch.bfloat16 when Q, K, V and O are all bf16, else torch.float16 (whose checks reject any other dtype)."""
    dts = [t.dtype for t in (Q, K, V, O)]
    if torch.bfloat16 not in dts:
        return torch.float16
    if any(d != torch.bfloat16 for d in dts):
        raise RuntimeError("leetcuda_b200.flash_attn: Q, K, V and O must share one dtype (all fp16 or all bf16), got "
                           + ", ".join(str(d).replace("torch.", "") for d in dts))
    return torch.bfloat16


_FP8_DTYPES = tuple(getattr(torch, n) for n in ("float8_e4m3fn", "float8_e5m2", "float8_e4m3fnuz", "float8_e5m2fnuz",
                                                 "float8_e8m0fnu") if hasattr(torch, n))


def _fp8_kv(Q, K, V, O):
    """Q's dtype when K and V are float8_e4m3fn (the fp8-K/V call), None when neither is an fp8 tensor."""
    dts = [t.dtype for t in (Q, K, V, O)]
    if not any(d in _FP8_DTYPES for d in dts):
        return None
    names = ", ".join(str(d).replace("torch.", "") for d in dts)
    if any(d in _FP8_DTYPES and d != torch.float8_e4m3fn for d in dts):
        raise RuntimeError(f"leetcuda_b200.flash_attn: fp8 K/V must be float8_e4m3fn (float8_e5m2 and the other fp8 "
                           f"formats are not supported), got Q, K, V, O = {names}")
    if Q.dtype in _FP8_DTYPES or O.dtype in _FP8_DTYPES:
        raise RuntimeError(f"leetcuda_b200.flash_attn: Q and O must be fp16 or bf16 (fp8 is for K and V only), "
                           f"got Q, K, V, O = {names}")
    if K.dtype != V.dtype:
        raise RuntimeError(f"leetcuda_b200.flash_attn: K and V must share one dtype (both float8_e4m3fn), "
                           f"got K {K.dtype}, V {V.dtype}".replace("torch.", ""))
    if Q.dtype != O.dtype or Q.dtype not in (torch.float16, torch.bfloat16):
        raise RuntimeError(f"leetcuda_b200.flash_attn: with fp8 K/V, Q and O must both be fp16 or both bf16, "
                           f"got Q {Q.dtype}, O {O.dtype}".replace("torch.", ""))
    return Q.dtype


def _placement(*tensors):
    for t in tensors:
        if not t.is_cuda:
            raise RuntimeError("leetcuda_b200.flash_attn: tensors must be CUDA tensors (no CPU path)")
        if not t.is_contiguous():
            raise RuntimeError("leetcuda_b200.flash_attn: tensors must be contiguous")


def _check(Q, K, V, O, v_transposed):
    # reference: CHECK_TORCH_TENSOR_DTYPE / _SHAPE (kernels/flash-attn/utils/utils.h:137-147): one length N for all
    B, H, N, _, D, _ = _shapes(Q, K, V, O, v_transposed, same_length=True)
    _placement(Q, K, V, O)
    return B, H, N, D


def fmha_fwd(Q, K, V, O, *, v_transposed: bool = False, scale: float = 0.0, lse=None, causal: bool = False,
             num_splits: int = 1, seqlens_q=None, seqlens_k=None, block_table=None, k_scale: float = 1.0,
             v_scale: float = 1.0) -> None:
    """``O = softmax(Q K^T * scale) V`` on the current CUDA stream of ``Q``'s device.

    Q, O are ``[B,H,Nq,D]``; K is ``[B,Hkv,Nk,D]`` and V ``[B,Hkv,Nk,D]`` (or ``[B,Hkv,D,Nk]`` with ``v_transposed``),
    where Nk may differ from Nq and Hkv may be any divisor of H: grouped-query attention, query head h reading K/V head
    ``h // (H // Hkv)`` as torch SDPA's ``enable_gqa`` does (Hkv = 1 is multi-query attention).  ``lse`` (optional,
    fp32 ``[B,H,Nq]`` CUDA tensor) receives ``ln sum_j exp(scale * q_i . k_j)`` per query row — the statistic
    ``merge_attn_states`` needs to combine results over disjoint key ranges.

    ``causal=True`` masks key j for query i when ``j > i + (Nk - Nq)``: the diagonal is aligned bottom-right as in
    FlashAttention-2 (the queries are the last Nq positions of the key sequence).  This is not torch SDPA's
    ``is_causal`` when Nq != Nk, which aligns it top-left.  Rows with no visible key (Nq > Nk) get O = 0, lse = -inf.

    ``num_splits`` cuts the keys of every CTA into that many ranges that run in parallel and are combined in fp32
    (split-KV, ``b200_fmha_fwd_f16_gqa``): 1 (the default) does not split, 0 lets the library choose from the shapes
    and the GPU's SM count — the choice for decoding (small Nq, long Nk), where an unsplit grid leaves most SMs idle.
    At most ``_capi.FMHA_MAX_SPLITS``.

    ``seqlens_q`` / ``seqlens_k`` (int32 contiguous CUDA tensors ``[B]`` on Q's device) give every sequence its own
    number of queries and keys inside the padded Q / K / V (``b200_fmha_fwd_f16_seqlens``): sequence b uses query rows
    ``0 .. clamp(seqlens_q[b], 0, Nq) - 1`` and key rows ``0 .. clamp(seqlens_k[b], 0, Nk) - 1``; keys past that
    contribute nothing whatever they hold, the causal diagonal is per sequence, and padded query rows get O = 0,
    lse = -inf.  The lengths are read on the GPU only (no host synchronisation), so a captured CUDA graph replays with
    whatever lengths the tensors hold.  None means Nq resp. Nk for every sequence; natural V only.

    ``block_table`` (int32 contiguous CUDA tensor ``[B, max_pages_per_seq]`` on Q's device) makes K and V paged KV-cache
    pools ``[num_pages, page_size, Hkv, D]`` (``b200_fmha_fwd_f16_paged``, the layout of FlashAttention's
    ``flash_attn_with_kvcache(block_table=...)``): key t of sequence b is row ``t % page_size`` of page
    ``block_table[b, t // page_size]``.  The call is then the ``seqlens_q`` / ``seqlens_k`` call on a padded cache of
    ``Nk = max_pages_per_seq * page_size`` keys, bit for bit, without gathering the pages.  Table entries past a
    sequence's last used page are never read (pad with -1 or stale ids); pages may be shared between sequences.  The
    table is read on the GPU only, so a captured graph replays with whatever tables and lengths the tensors hold.
    page_size must be a power of two >= 16; natural V only.

    Q, K, V and O are all fp16 or all bf16 (``torch.bfloat16``: ``b200_fmha_fwd_bf16_seqlens`` / ``_paged``, every option
    above but ``v_transposed``; lse stays fp32).  A bf16 call rounds P and O to bf16 where an fp16 one rounds them to fp16
    and is otherwise the same computation; a bf16 call without lengths runs the per-sequence-length kernel with every
    sequence at Nq / Nk.

    K and V may also be ``torch.float8_e4m3fn`` (an fp8 KV cache, dense, per-sequence or paged) with Q and O both fp16
    or both bf16 (``b200_fmha_fwd_{f16,bf16}_fp8kv_seqlens`` / ``_paged``): the call computes
    ``softmax(scale * Q (k_scale * K)^T) (v_scale * V)`` with every option above but ``v_transposed``.  ``k_scale`` and
    ``v_scale`` are per-tensor fp32 scales (finite, > 0; default 1) of the dequantisation ``x = scale * code``.  K and V
    are widened exactly to Q's type on the GPU, k_scale is folded into the softmax scale (fp32(scale * k_scale)) and
    v_scale multiplies the normalised O before its one rounding, so with v_scale = 1 the call is bit for bit the fp16 /
    bf16 seqlens or paged call on ``K.to(Q.dtype)``, ``V.to(Q.dtype)`` with that folded scale.  Scales other than 1
    are rejected with K and V that are not fp8."""
    fp8 = _fp8_kv(Q, K, V, O)
    if fp8 is not None:
        if v_transposed:
            raise RuntimeError("leetcuda_b200.flash_attn: transposed V is not supported with fp8 K/V "
                               "(v_transposed=True with float8_e4m3fn tensors)")
        scales = (float(k_scale), float(v_scale))
        _fmha_lens(Q, K, V, O, False, scale, lse, causal, num_splits, seqlens_q, seqlens_k, block_table, fp8, scales)
        return
    if k_scale != 1.0 or v_scale != 1.0:
        raise RuntimeError(f"leetcuda_b200.flash_attn: k_scale / v_scale apply to fp8 (float8_e4m3fn) K and V only, "
                           f"got k_scale={k_scale!r}, v_scale={v_scale!r} with K {K.dtype}, V {V.dtype}"
                           .replace("torch.", ""))
    dtype = _element_type(Q, K, V, O)
    if dtype == torch.bfloat16 and v_transposed:
        raise RuntimeError("leetcuda_b200.flash_attn: transposed V is fp16 only (v_transposed=True with bf16 tensors)")
    if block_table is not None or seqlens_q is not None or seqlens_k is not None or dtype == torch.bfloat16:
        _fmha_lens(Q, K, V, O, v_transposed, scale, lse, causal, num_splits, seqlens_q, seqlens_k, block_table, dtype)
        return
    B, H, Nq, Nk, D, Hkv = _shapes(Q, K, V, O, v_transposed, same_length=False, grouped=True)
    _check_lengths(Q, B, H, Nq, num_splits, lse, None, None)
    _placement(Q, K, V, O, *(() if lse is None else (lse,)))
    _run(Q, K, V, O, B, H, Nq, Nk, D, v_transposed, scale, lse, causal, Hkv, num_splits)


def _fmha_lens(Q, K, V, O, v_transposed, scale, lse, causal, num_splits, seqlens_q, seqlens_k, block_table,
               dtype=torch.float16, fp8_scales=None) -> None:
    """The seqlens call (``b200_fmha_fwd_*_seqlens``), or with ``block_table`` the paged one (``..._paged``)."""
    paged = block_table is not None
    if v_transposed:
        raise RuntimeError("leetcuda_b200.flash_attn: block_table takes natural V pools [num_pages,page_size,Hkv,D] "
                           "only (v_transposed=True is not supported with a block table)" if paged else
                           "leetcuda_b200.flash_attn: seqlens_q / seqlens_k take natural V [B,Hkv,Nk,D] only "
                           "(v_transposed=True is not supported with lengths)")
    if paged:
        if fp8_scales is None:
            _check_dtype(Q, K, V, O, dtype)
        if Q.dim() != 4 or tuple(O.shape) != tuple(Q.shape):
            raise RuntimeError("Tensor size mismatch!")
        B, H, Nq, D = Q.shape
        num_pages, page_size, Hkv = _check_pool("leetcuda_b200.flash_attn", K, V, D, H, "K", "V")
    else:
        B, H, Nq, Nk, D, Hkv = _shapes(Q, K, V, O, False, same_length=False, grouped=True, dtype=dtype,
                                       fp8=fp8_scales is not None)
    _check_lengths(Q, B, H, Nq, num_splits, lse, seqlens_q, seqlens_k)
    if paged:
        _check_block_table("leetcuda_b200.flash_attn", block_table, B, Q, "Q's")
    _placement(Q, K, V, O, *(() if lse is None else (lse,)))
    lens = [None if seqlens_q is None else seqlens_q.data_ptr(), None if seqlens_k is None else seqlens_k.data_ptr()]
    args = [Q.data_ptr(), K.data_ptr(), V.data_ptr(), O.data_ptr(), None if lse is None else lse.data_ptr()]
    if paged:
        args += [block_table.data_ptr()] + lens + [B, H, Hkv, Nq, num_pages, page_size, block_table.shape[1], D]
    else:
        args += lens + [B, H, Hkv, Nq, Nk, D]
    args += [int(bool(causal)), int(num_splits), float(scale)]
    name = "b200_fmha_fwd_bf16" if dtype == torch.bfloat16 else "b200_fmha_fwd_f16"
    if fp8_scales is not None:
        name += "_fp8kv"
        args += list(fp8_scales)
    _call_on_device(getattr(_capi.lib(), name + ("_paged" if paged else "_seqlens")), args, Q.device.index)


def _check_lengths(Q, B, H, Nq, num_splits, lse, seqlens_q, seqlens_k) -> None:
    """num_splits, lse and the length arrays of the seqlens and paged calls."""
    if isinstance(num_splits, bool) or not isinstance(num_splits, int) or not 0 <= num_splits <= _capi.FMHA_MAX_SPLITS:
        raise RuntimeError(f"leetcuda_b200.flash_attn: num_splits must be an int in 0 .. {_capi.FMHA_MAX_SPLITS}, "
                           f"got {num_splits!r}")
    if lse is not None and (lse.dtype != torch.float32 or tuple(lse.shape) != (B, H, Nq)):
        raise RuntimeError("leetcuda_b200.flash_attn: lse must be a contiguous fp32 CUDA tensor [B,H,Nq]")
    for name, t in (("seqlens_q", seqlens_q), ("seqlens_k", seqlens_k)):
        if t is None:
            continue
        if not isinstance(t, torch.Tensor) or t.dtype != torch.int32 or tuple(t.shape) != (B,) or not t.is_cuda \
                or not t.is_contiguous() or t.device != Q.device:
            raise RuntimeError(f"leetcuda_b200.flash_attn: {name} must be an int32 contiguous CUDA tensor [B] = [{B}] "
                               f"on Q's device")


def _check_pool(who, K, V, D, H, k_name, v_name):
    """(num_pages, page_size, Hkv) of the paged K/V pools K and V [num_pages, page_size, Hkv, D]."""
    if K.dim() != 4 or tuple(K.shape) != tuple(V.shape) or K.shape[3] != D or K.shape[2] < 1 or H % K.shape[2] \
            or K.shape[0] < 1:
        raise RuntimeError(f"{who}: with block_table, {k_name} and {v_name} must be pools "
                           f"[num_pages, page_size, Hkv, D] of the same shape, with D = {D} and Hkv dividing H = {H}")
    num_pages, page_size, Hkv, _ = K.shape
    if page_size < 16 or page_size & (page_size - 1):
        raise RuntimeError(f"{who}: page_size ({k_name}.shape[1]) must be a power of two >= 16, got {page_size}")
    return num_pages, page_size, Hkv


def _check_block_table(who, t, B, q, q_name) -> None:
    if not isinstance(t, torch.Tensor) or t.dtype != torch.int32 or t.dim() != 2 or t.shape[0] != B \
            or t.shape[1] < 1 or not t.is_cuda or not t.is_contiguous() or t.device != q.device:
        raise RuntimeError(f"{who}: block_table must be an int32 contiguous CUDA tensor "
                           f"[B, max_pages_per_seq] = [{B}, >= 1] on {q_name} device")


def fmha_varlen_fwd(q, k, v, o, cu_seqlens_q, cu_seqlens_k, max_seqlen_q: int, max_seqlen_k: int, *,
                    scale: float = 0.0, causal: bool = False, lse=None, block_table=None, seqused_k=None,
                    num_splits: int = 1, v_transposed: bool = False, rms_g: float = 0.0) -> None:
    """Packed variable-length attention, FlashAttention's ``flash_attn_varlen_func`` layout, on the current CUDA stream
    of ``q``'s device (``b200_fmha_fwd_{f16,bf16}_varlen``; with ``block_table``: ``..._varlen_paged``).

    ``q``, ``o`` are ``[total_q, H, D]`` and ``k``, ``v`` ``[total_k, Hkv, D]``, fp16 or bf16 (one dtype for all four),
    contiguous, with Hkv dividing H (query head h reads K/V head ``h // (H // Hkv)``).  ``cu_seqlens_q`` and
    ``cu_seqlens_k`` are int32 contiguous CUDA tensors ``[B + 1]``: sequence b has
    ``Lq_b = clamp(cu_seqlens_q[b+1] - cu_seqlens_q[b], 0, max_seqlen_q)`` queries at rows ``cu_seqlens_q[b] + t`` and
    ``Lk_b = clamp(cu_seqlens_k[b+1] - cu_seqlens_k[b], 0, max_seqlen_k)`` keys at rows ``cu_seqlens_k[b] + t``.
    ``causal=True`` masks key j for query i when ``j > i + (Lk_b - Lq_b)`` (bottom-right, per sequence, as
    ``fmha_fwd(seqlens_q=, seqlens_k=)``).  ``lse`` (optional) is fp32 ``[H, total_q]``, the layout of
    ``merge_attn_states``, so the O and lse of two calls over disjoint keys merge without a reshape.

    ``block_table`` (int32 ``[B, max_pages_per_seq]``) makes ``k`` and ``v`` paged pools
    ``[num_pages, page_size, Hkv, D]`` as in ``fmha_fwd(block_table=)``: then ``cu_seqlens_k`` must be None,
    ``seqused_k`` (int32 ``[B]``) gives ``Lk_b = clamp(seqused_k[b], 0, max_pages_per_seq * page_size)``,
    ``max_seqlen_k`` is ignored, and key t of sequence b is row ``t % page_size`` of page ``block_table[b][t // page_size]``.

    Only rows ``cu_seqlens_q[b] + t`` with ``t < Lq_b`` inside ``o`` are written: rows of ``o`` and columns of ``lse``
    that belong to no sequence keep their contents.  Rows without a visible key get O = 0 and lse = -inf.  Keys of the
    next sequence contribute nothing whatever they hold.  Offsets, lengths and tables are read on the GPU only (no host
    synchronisation), so a captured CUDA graph replays with new values written into the same tensors.  The results are
    bit for bit ``fmha_fwd(seqlens_q=, seqlens_k=, num_splits=1)`` (or the ``block_table`` call) on padded copies.

    Every query head gets ``ceil(max_seqlen_q / 128)`` query tiles of its own (64-row tiles for D > 128).  A batch of
    one-token decode rows therefore fills one row of every tile: use ``fmha_fwd`` with ``seqlens_q`` / ``block_table``
    for decoding.  Not supported, and rejected by name: ``num_splits`` other than 1, fp8 K/V, ``v_transposed`` and the
    fused RMS norm (``rms_g``)."""
    if isinstance(num_splits, bool) or num_splits != 1:
        raise RuntimeError(f"leetcuda_b200.flash_attn.fmha_varlen_fwd: num_splits={num_splits!r} is not supported "
                           f"(varlen runs unsplit: num_splits must be 1)")
    if v_transposed:
        raise RuntimeError("leetcuda_b200.flash_attn.fmha_varlen_fwd: v_transposed=True is not supported (natural V "
                           "[total_k, Hkv, D] only)")
    if rms_g:
        raise RuntimeError(f"leetcuda_b200.flash_attn.fmha_varlen_fwd: the fused RMS norm (rms_g={rms_g!r}) is not "
                           f"supported with varlen")
    who = "leetcuda_b200.flash_attn.fmha_varlen_fwd"
    for name, t in (("q", q), ("k", k), ("v", v), ("o", o)):
        if not isinstance(t, torch.Tensor):
            raise RuntimeError(f"{who}: {name} must be a torch.Tensor")
    if any(t.dtype in _FP8_DTYPES for t in (q, k, v, o)):
        raise RuntimeError(f"{who}: fp8 K/V is not supported with varlen (use fmha_fwd with float8_e4m3fn K/V)")
    dts = {t.dtype for t in (q, k, v, o)}
    if len(dts) != 1 or q.dtype not in (torch.float16, torch.bfloat16):
        raise RuntimeError(f"{who}: q, k, v and o must share one dtype, fp16 or bf16, got "
                           + ", ".join(str(t.dtype).replace("torch.", "") for t in (q, k, v, o)))
    if q.dim() != 3 or tuple(o.shape) != tuple(q.shape):
        raise RuntimeError(f"{who}: q and o must be [total_q, H, D] of one shape, got q {tuple(q.shape)}, "
                           f"o {tuple(o.shape)}")
    total_q, H, D = q.shape
    paged = block_table is not None
    for name, x in (("max_seqlen_q", max_seqlen_q), ("max_seqlen_k", max_seqlen_k)):
        if isinstance(x, bool) or not isinstance(x, int):
            raise RuntimeError(f"{who}: {name} must be an int, got {x!r}")
    if paged:
        if cu_seqlens_k is not None:
            raise RuntimeError(f"{who}: with block_table, cu_seqlens_k must be None (seqused_k gives the keys)")
        num_pages, page_size, Hkv = _check_pool(who, k, v, D, H, "k", "v")
    else:
        if seqused_k is not None:
            raise RuntimeError(f"{who}: seqused_k needs block_table (packed K/V take their lengths from cu_seqlens_k)")
        if k.dim() != 3 or tuple(k.shape) != tuple(v.shape) or k.shape[2] != D or k.shape[1] < 1 or H % k.shape[1]:
            raise RuntimeError(f"{who}: k and v must be [total_k, Hkv, D] of one shape, with D = {D} and Hkv dividing "
                               f"H = {H}, got k {tuple(k.shape)}, v {tuple(v.shape)}")
        total_k, Hkv, _ = k.shape
    if lse is not None and (not isinstance(lse, torch.Tensor) or lse.dtype != torch.float32
                            or tuple(lse.shape) != (H, total_q)):
        raise RuntimeError(f"{who}: lse must be a contiguous fp32 CUDA tensor [H, total_q] = [{H}, {total_q}]")
    if not isinstance(cu_seqlens_q, torch.Tensor) or cu_seqlens_q.dim() != 1 or cu_seqlens_q.shape[0] < 2:
        raise RuntimeError(f"{who}: cu_seqlens_q must be an int32 contiguous CUDA tensor [B + 1] (B >= 1) on q's device")
    B = cu_seqlens_q.shape[0] - 1
    if paged:
        _check_block_table(who, block_table, B, q, "q's")
    arrays = [("cu_seqlens_q", cu_seqlens_q, B + 1)]
    arrays += [("seqused_k", seqused_k, B)] if paged else [("cu_seqlens_k", cu_seqlens_k, B + 1)]
    for on_device in (False, True):   # every array's type and shape first, then where it lives
        for name, t, n in arrays:
            if not (isinstance(t, torch.Tensor) and t.dtype == torch.int32 and tuple(t.shape) == (n,)
                    and t.is_contiguous()) or on_device and not (t.is_cuda and t.device == q.device):
                raise RuntimeError(f"{who}: {name} must be an int32 contiguous CUDA tensor [{n}] on q's device")
    for name, t in (("q", q), ("k", k), ("v", v), ("o", o)) + ((("lse", lse),) if lse is not None else ()):
        if not t.is_cuda or t.device != q.device:
            raise RuntimeError(f"{who}: {name} must be a CUDA tensor on q's device (no CPU path)")
        if not t.is_contiguous():
            raise RuntimeError(f"{who}: {name} must be contiguous")
    name = "b200_fmha_fwd_bf16_varlen" if q.dtype == torch.bfloat16 else "b200_fmha_fwd_f16_varlen"
    lse_ptr = None if lse is None else lse.data_ptr()
    if paged:
        args = [q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), lse_ptr, cu_seqlens_q.data_ptr(),
                seqused_k.data_ptr(), block_table.data_ptr(), B, H, Hkv, total_q, int(max_seqlen_q), num_pages,
                page_size, block_table.shape[1], D, int(bool(causal)), float(scale)]
        name += "_paged"
    else:
        args = [q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr(), lse_ptr, cu_seqlens_q.data_ptr(),
                cu_seqlens_k.data_ptr(), B, H, Hkv, total_q, total_k, int(max_seqlen_q), int(max_seqlen_k), D,
                int(bool(causal)), float(scale)]
    _call_on_device(getattr(_capi.lib(), name), args, q.device.index)


def kvcache_append(k, v, k_cache, v_cache, cache_seqlens, *, block_table=None, q=None, q_out=None, rotary_cos=None,
                   rotary_sin=None, rotary_interleaved: bool = False, k_scale: float = 1.0, v_scale: float = 1.0,
                   seqlens_out=None) -> None:
    """Append n_new tokens per sequence to a KV cache, with rotary embedding, in one launch on the current CUDA stream of
    ``k``'s device (``b200_kvcache_append_{f16,bf16}``; with ``block_table``: ``..._paged``).  The write half of
    FlashAttention's ``flash_attn_with_kvcache`` and vLLM's ``reshape_and_cache_flash``.

    ``k``, ``v`` are ``[B, Hkv, n_new, D]`` fp16 or bf16.  ``cache_seqlens`` (int32 ``[B]``) gives the tokens sequence b
    already holds, ``L_b = clamp(cache_seqlens[b], 0, capacity)``; new token t goes to position ``L_b + t``.  Dense
    ``k_cache``, ``v_cache`` are ``[B, Hkv, Nk, D]`` (capacity Nk, the layout ``fmha_fwd(seqlens_k=)`` reads); with
    ``block_table`` (int32 ``[B, max_pages_per_seq]``) they are pools ``[num_pages, page_size, Hkv, D]`` (capacity
    ``max_pages_per_seq * page_size``) and position p is row ``p % page_size`` of page ``block_table[b, p // page_size]``.
    Tokens past capacity, and tokens whose table entry is outside ``[0, num_pages)``, are not written; no other cache
    byte changes.  Two sequences writing the same row of a shared page race (not detected).

    The cache has k's dtype, or is ``torch.float8_e4m3fn``: then it receives ``(x.float() / scale).clamp(-448, 448)``
    in e4m3 (round to nearest even), x the fp16 / bf16 value after rotary, k with ``k_scale`` and v with ``v_scale``
    (finite, > 0; exactly 1 for an fp16 / bf16 cache).

    ``rotary_cos``, ``rotary_sin`` (fp32 ``[rotary_len, rotary_dim / 2]``, ``rotary_len >= capacity + n_new``,
    ``rotary_dim`` a multiple of 16 up to D) rotate k (never v) at each token's position: pair i is ``(2i, 2i+1)`` with
    ``rotary_interleaved`` (GPT-J) and ``(i, i + rotary_dim / 2)`` without (NeoX / Llama), ``x0' = x0 cos - x1 sin``,
    ``x1' = x0 sin + x1 cos`` in fp32, rounded once; columns past rotary_dim are copied.  ``q`` (``[B, H, n_new, D]``) is
    rotated at the same positions into ``q_out`` (default: ``q`` itself, in place; otherwise a tensor that shares no
    memory with the others).  ``seqlens_out`` (int32 ``[B]``, not ``cache_seqlens``) receives ``min(L_b + n_new,
    capacity)``, the ``seqlens_k`` of the attention call.  Lengths and tables are read on the GPU only (no host
    synchronisation), so a captured CUDA graph replays with the values the tensors hold."""
    who = "leetcuda_b200.flash_attn.kvcache_append"
    _append(who, k, v, k_cache, v_cache, cache_seqlens, block_table, q, q_out, rotary_cos, rotary_sin,
            rotary_interleaved, k_scale, v_scale, seqlens_out)


def _append(who, k, v, k_cache, v_cache, cache_seqlens, block_table, q, q_out, rotary_cos, rotary_sin,
            rotary_interleaved, k_scale, v_scale, seqlens_out) -> None:
    named = (("k", k), ("v", v), ("k_cache", k_cache), ("v_cache", v_cache), ("cache_seqlens", cache_seqlens))
    opt = (("block_table", block_table), ("q", q), ("q_out", q_out), ("rotary_cos", rotary_cos),
           ("rotary_sin", rotary_sin), ("seqlens_out", seqlens_out))
    for name, t in named + opt:
        if (t is not None or name in dict(named)) and not isinstance(t, torch.Tensor):
            raise RuntimeError(f"{who}: {name} must be a torch.Tensor")
    if q_out is not None and q is None:
        raise RuntimeError(f"{who}: q_out needs q")
    if (rotary_cos is None) != (rotary_sin is None):
        raise RuntimeError(f"{who}: rotary_cos and rotary_sin must both be given or both be None")
    if k.dtype not in (torch.float16, torch.bfloat16) or v.dtype != k.dtype:
        raise RuntimeError(f"{who}: k and v must share one dtype, fp16 or bf16, got k {k.dtype}, v {v.dtype}"
                           .replace("torch.", ""))
    if k_cache.dtype != v_cache.dtype or k_cache.dtype not in (k.dtype, torch.float8_e4m3fn):
        raise RuntimeError(f"{who}: k_cache and v_cache must both have k's dtype or both be float8_e4m3fn, got "
                           f"k_cache {k_cache.dtype}, v_cache {v_cache.dtype} with k {k.dtype}".replace("torch.", ""))
    e4m3 = k_cache.dtype == torch.float8_e4m3fn
    if k.dim() != 4 or tuple(v.shape) != tuple(k.shape):
        raise RuntimeError(f"{who}: k and v must be [B, Hkv, n_new, D] of one shape, got k {tuple(k.shape)}, "
                           f"v {tuple(v.shape)}")
    B, Hkv, n_new, D = k.shape
    paged = block_table is not None
    if paged:
        if k_cache.dim() != 4 or tuple(v_cache.shape) != tuple(k_cache.shape) or tuple(k_cache.shape[2:]) != (Hkv, D):
            raise RuntimeError(f"{who}: with block_table, k_cache and v_cache must be pools [num_pages, page_size, Hkv, "
                               f"D] of one shape with Hkv = {Hkv}, D = {D}, got k_cache {tuple(k_cache.shape)}, "
                               f"v_cache {tuple(v_cache.shape)}")
        num_pages, page_size = k_cache.shape[:2]
        if page_size < 16 or page_size & (page_size - 1):
            raise RuntimeError(f"{who}: page_size (k_cache.shape[1]) must be a power of two >= 16, got {page_size}")
        t = block_table
        if t.dtype != torch.int32 or t.dim() != 2 or t.shape[0] != B or t.shape[1] < 1:
            raise RuntimeError(f"{who}: block_table must be an int32 contiguous CUDA tensor [B, max_pages_per_seq] = "
                               f"[{B}, >= 1] on k's device")
        capacity = t.shape[1] * page_size
    else:
        if k_cache.dim() != 4 or tuple(v_cache.shape) != tuple(k_cache.shape) or k_cache.shape[0] != B \
                or k_cache.shape[1] != Hkv or k_cache.shape[3] != D:
            raise RuntimeError(f"{who}: k_cache and v_cache must be [B, Hkv, Nk, D] of one shape with B = {B}, "
                               f"Hkv = {Hkv}, D = {D}, got k_cache {tuple(k_cache.shape)}, v_cache {tuple(v_cache.shape)}")
        capacity = k_cache.shape[2]
    H = Hkv
    if q is not None:
        if q.dtype != k.dtype or q.dim() != 4 or q.shape[0] != B or q.shape[2] != n_new or q.shape[3] != D \
                or q.shape[1] < 1 or q.shape[1] % max(Hkv, 1):
            raise RuntimeError(f"{who}: q must be [B, H, n_new, D] = [{B}, H, {n_new}, {D}] of k's dtype with Hkv = "
                               f"{Hkv} dividing H, got {tuple(q.shape)} {q.dtype}".replace("torch.", ""))
        H = q.shape[1]
        if q_out is None:
            q_out = q
        elif q_out.dtype != q.dtype or tuple(q_out.shape) != tuple(q.shape):
            raise RuntimeError(f"{who}: q_out must have q's shape and dtype")
    rotary_dim = rotary_len = 0
    if rotary_cos is not None:
        c, s = rotary_cos, rotary_sin
        if c.dtype != torch.float32 or s.dtype != torch.float32 or c.dim() != 2 or tuple(s.shape) != tuple(c.shape):
            raise RuntimeError(f"{who}: rotary_cos and rotary_sin must be fp32 [rotary_len, rotary_dim / 2] of one shape")
        rotary_len, rotary_dim = c.shape[0], 2 * c.shape[1]
        if rotary_dim < 16 or rotary_dim > D or rotary_dim % 16:
            raise RuntimeError(f"{who}: rotary_dim = 2 * rotary_cos.shape[1] = {rotary_dim} must be a multiple of 16 in "
                               f"16 .. D = {D}")
        if rotary_len < capacity + n_new:
            raise RuntimeError(f"{who}: rotary_cos.shape[0] = {rotary_len} must be >= capacity + n_new = "
                               f"{capacity + n_new} (the largest position a token can get, plus one)")
    elif rotary_interleaved:
        raise RuntimeError(f"{who}: rotary_interleaved needs rotary_cos and rotary_sin")
    for name, x in (("k_scale", k_scale), ("v_scale", v_scale)):
        x = float(x)
        if not (math.isfinite(x) and x > 0):
            raise RuntimeError(f"{who}: {name}={x!r} must be finite and > 0")
        if not e4m3 and x != 1.0:
            raise RuntimeError(f"{who}: {name}={x!r} must be 1 unless the cache is float8_e4m3fn")
    for name, t in (("cache_seqlens", cache_seqlens), ("seqlens_out", seqlens_out)):
        if t is not None and (t.dtype != torch.int32 or tuple(t.shape) != (B,)):
            raise RuntimeError(f"{who}: {name} must be an int32 contiguous CUDA tensor [B] = [{B}] on k's device")
    present = [(n, t) for n, t in named + opt if t is not None]
    for name, t in present:
        if not t.is_cuda or t.device != k.device:
            raise RuntimeError(f"{who}: {name} must be a CUDA tensor on k's device (no CPU path)")
        if not t.is_contiguous():
            raise RuntimeError(f"{who}: {name} must be contiguous")
    # every buffer the kernel writes shares no byte with another one; q_out may be q itself (rotated in place)
    present = [(n, t) for n, t in present if n != "q_out" and t is not None]
    if q_out is not None and q_out.data_ptr() != q.data_ptr():
        present.append(("q_out", q_out))
    for wname, w in present:
        if wname in ("k_cache", "v_cache", "q_out", "seqlens_out"):
            for name, t in present:
                if name != wname and _capi.overlaps(w, t):
                    raise RuntimeError(f"{who}: {wname} overlaps {name}")
    ptr = lambda t: None if t is None else t.data_ptr()   # noqa: E731
    cdt = _capi.DTYPE_E4M3 if e4m3 else (_capi.DTYPE_BF16 if k.dtype == torch.bfloat16 else _capi.DTYPE_F16)
    name = "b200_kvcache_append_bf16" if k.dtype == torch.bfloat16 else "b200_kvcache_append_f16"
    head = [k.data_ptr(), v.data_ptr(), k_cache.data_ptr(), v_cache.data_ptr()]
    mid = [cache_seqlens.data_ptr(), ptr(seqlens_out), ptr(q), ptr(q_out), ptr(rotary_cos), ptr(rotary_sin), B, H, Hkv,
           n_new]
    tail = [D, rotary_dim, rotary_len, int(bool(rotary_interleaved)), cdt, float(k_scale), float(v_scale)]
    if paged:
        args = head + [block_table.data_ptr()] + mid + [num_pages, page_size, block_table.shape[1]] + tail
        name += "_paged"
    else:
        args = head + mid + [capacity] + tail
    _call_on_device(getattr(_capi.lib(), name), args, k.device.index, "kvcache_append", headdim=False)


def fmha_fwd_kvcache(q, k_cache, v_cache, o, k, v, cache_seqlens, *, block_table=None, rotary_cos=None,
                     rotary_sin=None, rotary_interleaved: bool = False, causal: bool = False, scale: float = 0.0,
                     lse=None, num_splits: int = 1, k_scale: float = 1.0, v_scale: float = 1.0):
    """One decode or chunked-prefill step: append ``k``, ``v`` (``[B, Hkv, n_new, D]``) to the cache with
    ``kvcache_append`` (rotary on q and k at positions ``L_b + t``, e4m3 quantisation for a ``float8_e4m3fn`` cache,
    paging through ``block_table``), then attend ``q`` (``[B, H, n_new, D]``) over the cache with ``fmha_fwd``
    (``seqlens_k`` = the new lengths, ``seqlens_q`` = None so Nq = n_new, ``block_table``, ``k_scale`` / ``v_scale``),
    writing ``o``.  Returns the new lengths, int32 ``[B]``: ``min(L_b + n_new, capacity)``.

    The queries are the last n_new positions of each sequence, which is where the causal diagonal sits (bottom-right),
    and q is rotated at the same positions ``L_b + t`` as the keys, causal or not.  FlashAttention's
    ``flash_attn_with_kvcache`` rotates non-causal q at ``L_b`` for every t instead; with n_new = 1 the two agree.
    The rotated q goes into a new tensor (``q`` is not modified); without rotary tables ``q`` is used as it is.
    Two launches plus the attention's split combine if any (1 + 1 or 2).  ``k`` and ``v`` are required: attention over a
    cache without an append is ``fmha_fwd(seqlens_k=)``.  Everything is read on the GPU, with no host synchronisation,
    so the step can be captured in a CUDA graph."""
    who = "leetcuda_b200.flash_attn.fmha_fwd_kvcache"
    for name, t in (("q", q), ("o", o), ("k", k), ("v", v)):
        if not isinstance(t, torch.Tensor):
            raise RuntimeError(f"{who}: {name} must be a torch.Tensor (k and v are required)")
    if q.dim() != 4 or tuple(o.shape) != tuple(q.shape) or o.dtype != q.dtype:
        raise RuntimeError(f"{who}: o must have q's shape [B, H, n_new, D] and dtype")
    if q.shape[3] > 1024:
        raise RuntimeError(f"{who}: headdim not support! (D={q.shape[3]} > 1024)")
    if k.dim() != 4 or q.dtype != k.dtype or (q.shape[0], q.shape[2], q.shape[3]) != (k.shape[0], k.shape[2], k.shape[3]) \
            or k.shape[1] < 1 or q.shape[1] % k.shape[1]:
        raise RuntimeError(f"{who}: q must be [B, H, n_new, D] of k's dtype, k [B, Hkv, n_new, D] with Hkv dividing H, "
                           f"got q {tuple(q.shape)} {q.dtype}, k {tuple(k.shape)} {k.dtype}".replace("torch.", ""))
    _check_lengths(q, q.shape[0], q.shape[1], q.shape[2], num_splits, lse, None, None)
    if isinstance(cache_seqlens, torch.Tensor) and cache_seqlens.dim() == 1:
        new_lens = torch.empty(cache_seqlens.shape[0], dtype=torch.int32, device=cache_seqlens.device)
    else:
        new_lens = None   # _append rejects it
    q_rot = torch.empty_like(q) if rotary_cos is not None else None
    _append(who, k, v, k_cache, v_cache, cache_seqlens, block_table, None if q_rot is None else q, q_rot, rotary_cos,
            rotary_sin, rotary_interleaved, k_scale, v_scale, new_lens)
    kw = dict(scale=scale, lse=lse, causal=causal, num_splits=num_splits, seqlens_k=new_lens, block_table=block_table)
    if k_cache.dtype == torch.float8_e4m3fn:
        kw.update(k_scale=k_scale, v_scale=v_scale)
    fmha_fwd(q if q_rot is None else q_rot, k_cache, v_cache, o, **kw)
    return new_lens


def _call_on_device(fn, args, idx, label="fmha_fwd", headdim=True) -> None:
    """fn(*args, stream) on device idx's current stream; headdim: B200_ENOTSUP raises the reference's text."""
    if torch.cuda.current_device() != idx:
        with torch.cuda.device(idx):
            rc = fn(*args, _capi.raw_stream(idx))
    else:
        rc = fn(*args, _capi.raw_stream(idx))
    if headdim and rc == -3:  # B200_ENOTSUP: the reference throws exactly this text (flash_attn_mma_split_q.cu:793)
        raise RuntimeError("headdim not support!")
    _capi.check(rc, label)


def _fmha_one_length(Q, K, V, O, v_transposed=False) -> None:
    """The reference ops: q, k, v, o of one sequence length ("Tensor size mismatch!" otherwise), no mask."""
    B, H, N, D = _check(Q, K, V, O, v_transposed)
    _run(Q, K, V, O, B, H, N, N, D, v_transposed, 0.0, None, False)


def _run(Q, K, V, O, B, H, Nq, Nk, D, v_transposed, scale, lse, causal, Hkv=None, num_splits=1) -> None:
    args = [Q.data_ptr(), K.data_ptr(), V.data_ptr(), O.data_ptr()]
    if (Hkv is not None and Hkv != H) or num_splits != 1:
        fn = _capi.lib().b200_fmha_fwd_f16_gqa
        args += [None if lse is None else lse.data_ptr(), B, H, Hkv, Nq, Nk, D, int(v_transposed), int(bool(causal)),
                 int(num_splits), float(scale)]
    elif causal or Nk != Nq:
        fn = _capi.lib().b200_fmha_fwd_f16_kv
        args += [None if lse is None else lse.data_ptr(), B, H, Nq, Nk, D, int(v_transposed), int(bool(causal)),
                 float(scale)]
    else:
        if lse is not None:
            fn = _capi.lib().b200_fmha_fwd_f16_lse
            args.append(lse.data_ptr())
        else:
            fn = _capi.lib().b200_fmha_fwd_f16
        args += [B, H, Nq, D, int(v_transposed), float(scale)]
    _call_on_device(fn, args, Q.device.index)


def fmha_host(Q, K, V, O, *, v_transposed: bool = False, scale: float = 0.0) -> None:
    """Host-buffer entry point (``b200_fmha_fwd_f16_host``): ``Q``, ``K``, ``V``, ``O`` are CPU fp16 tensors
    (pinned for full PCIe bandwidth).  The call uploads the inputs, runs the kernel on the current device and
    downloads ``O``, pipelined over (batch x head) chunks; it returns when ``O`` is complete."""
    for t in (Q, K, V, O):
        if t.dtype != torch.float16:
            raise RuntimeError("values must be torch::kHalf")
        if t.is_cuda or not t.is_contiguous():
            raise RuntimeError("leetcuda_b200.fmha_host: tensors must be contiguous host tensors")
    B, H, N, D = Q.shape
    want_v = (B, H, D, N) if v_transposed else (B, H, N, D)
    if tuple(K.shape) != (B, H, N, D) or tuple(O.shape) != (B, H, N, D) or tuple(V.shape) != want_v:
        raise RuntimeError("Tensor size mismatch!")
    idx = torch.cuda.current_device()
    _call_on_device(_capi.lib().b200_fmha_fwd_f16_host, [Q.data_ptr(), K.data_ptr(), V.data_ptr(), O.data_ptr(), B, H,
                    N, D, int(v_transposed), float(scale)], idx, "fmha_host")


def _make(name: str):
    vt = name in V_TRANSPOSED_OPS

    def op(Q, K, V, O, stages: int = 1) -> None:
        _fmha_one_length(Q, K, V, O, v_transposed=vt)
    op.__name__ = op.__qualname__ = name
    op.__doc__ = (f"{name}(Q, K, V, O, stages) -> None  "
                  f"[V is {'[B,H,D,N]' if vt else '[B,H,N,D]'}; stages ignored; sm_90a fused kernel]")
    return op


for _n in OP_NAMES:
    globals()[_n] = _make(_n)


def flash_attn_cute(Q, K, V, O) -> None:
    """reference: kernels/flash-attn/cutlass/flash_attn_cute.cu:496-524."""
    _fmha_one_length(Q, K, V, O)


__all__ = OP_NAMES + ["flash_attn_cute", "fmha_fwd", "fmha_varlen_fwd", "fmha_host", "kvcache_append",
           "fmha_fwd_kvcache", "OP_NAMES", "V_TRANSPOSED_OPS"]
