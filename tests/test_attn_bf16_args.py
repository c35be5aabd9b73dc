"""Argument checks of the bf16 attention entries and of flash_attn.fmha_fwd on bf16 tensors: rejected on the host, before
any CUDA call (no GPU needed).  The C entries b200_fmha_fwd_bf16_seqlens / _paged run exactly the checks, and give
exactly the messages, of their f16 counterparts: the argument tables of test_attn_seqlens_args / test_attn_paged_args
are replayed against them."""
import pytest
import torch

import test_attn_paged_args as PA
import test_attn_seqlens_args as SA
from leetcuda_b200 import _capi, flash_attn


def _table(test):
    return [m for m in test.pytestmark if m.name == "parametrize"][0].args[1]


class _Bf16Entries:
    """The f16 module's lib with its f16 entry answered by the bf16 one."""

    def __init__(self, lib):
        self.b200_fmha_fwd_f16_seqlens = lib.b200_fmha_fwd_bf16_seqlens
        self.b200_fmha_fwd_f16_paged = lib.b200_fmha_fwd_bf16_paged


@pytest.mark.parametrize("kw,text", _table(SA.test_c_argument_checks))
def test_c_seqlens_checks_match_f16(built_lib, kw, text):
    assert SA._sl(_Bf16Entries(built_lib), **kw) == SA._sl(built_lib, **kw) == -1
    f16 = _capi.last_error()
    SA._sl(_Bf16Entries(built_lib), **kw)
    assert _capi.last_error() == f16 and f16.startswith("fmha_seqlens: ") and text in f16


@pytest.mark.parametrize("kw,text", _table(PA.test_c_argument_checks))
def test_c_paged_checks_match_f16(built_lib, kw, text):
    assert PA._pg(_Bf16Entries(built_lib), **kw) == PA._pg(built_lib, **kw) == -1
    f16 = _capi.last_error()
    PA._pg(_Bf16Entries(built_lib), **kw)
    assert _capi.last_error() == f16 and f16.startswith("fmha_paged: ") and text in f16


@pytest.mark.parametrize("D", [100, 1032])
def test_c_head_dim(built_lib, D):
    assert SA._sl(_Bf16Entries(built_lib), D=D, splits=0) == -3
    assert _capi.last_error().startswith("fmha_seqlens: headdim not support!")
    assert PA._pg(_Bf16Entries(built_lib), D=D, splits=0) == -3
    assert _capi.last_error().startswith("fmha_paged: headdim not support!")


def _t(*shape, dtype=torch.bfloat16):
    return torch.zeros(*shape, dtype=dtype)


_FP = {"fp16": torch.float16, "bf16": torch.bfloat16, "fp32": torch.float32}


@pytest.mark.parametrize("dts", ["bf16 fp16 bf16 bf16", "fp16 bf16 fp16 fp16", "bf16 bf16 bf16 fp32",
                                 "bf16 bf16 fp16 bf16", "fp32 bf16 bf16 bf16"])
@pytest.mark.parametrize("paged", [False, True], ids=["contiguous", "paged"])
def test_python_rejects_mixed_dtypes(dts, paged):
    q, k, v, o = (_FP[d] for d in dts.split())
    kv = (40, 16, 2, 64) if paged else (2, 2, 300, 64)
    extra = dict(block_table=torch.zeros(2, 8, dtype=torch.int32)) if paged else {}
    with pytest.raises(RuntimeError, match="must share one dtype"):
        flash_attn.fmha_fwd(_t(2, 8, 5, 64, dtype=q), _t(*kv, dtype=k), _t(*kv, dtype=v), _t(2, 8, 5, 64, dtype=o),
                            **extra)


def test_python_fp32_still_reads_khalf():
    """Without bf16 among them the fp16 checks and texts are unchanged (test_attn_paged_args expects this one)."""
    pool = _t(40, 16, 2, 64, dtype=torch.float32)
    with pytest.raises(RuntimeError, match="values must be torch::kHalf"):
        flash_attn.fmha_fwd(_t(2, 8, 5, 64, dtype=torch.float16), pool, pool, _t(2, 8, 5, 64, dtype=torch.float16),
                            block_table=torch.zeros(2, 8, dtype=torch.int32))


@pytest.mark.parametrize("extra", [{}, dict(causal=True, num_splits=0),
                                   dict(seqlens_k=torch.zeros(2, dtype=torch.int32)),
                                   dict(block_table=torch.zeros(2, 8, dtype=torch.int32))],
                         ids=["dense", "causal-auto", "seqlens", "paged"])
def test_python_rejects_transposed_v(extra):
    k = _t(40, 16, 2, 64) if "block_table" in extra else _t(2, 2, 300, 64)
    with pytest.raises(RuntimeError, match="transposed V is fp16 only"):
        flash_attn.fmha_fwd(_t(2, 8, 5, 64), k, _t(2, 2, 64, 300), _t(2, 8, 5, 64), v_transposed=True, **extra)


def test_python_bf16_keeps_the_other_checks():
    with pytest.raises(RuntimeError, match="Tensor size mismatch!"):
        flash_attn.fmha_fwd(_t(2, 8, 5, 64), _t(2, 2, 300, 64), _t(2, 2, 300, 64), _t(2, 8, 6, 64))
    with pytest.raises(RuntimeError, match="num_splits must be an int"):
        flash_attn.fmha_fwd(_t(2, 8, 5, 64), _t(2, 2, 300, 64), _t(2, 2, 300, 64), _t(2, 8, 5, 64), num_splits=65)
    with pytest.raises(RuntimeError, match=r"lse must be .*\[B,H,Nq\]"):
        flash_attn.fmha_fwd(_t(2, 8, 5, 64), _t(2, 2, 300, 64), _t(2, 2, 300, 64), _t(2, 8, 5, 64),
                            lse=torch.zeros(2, 8, 6))
    with pytest.raises(RuntimeError, match="tensors must be CUDA tensors"):
        flash_attn.fmha_fwd(_t(2, 8, 5, 64), _t(2, 2, 300, 64), _t(2, 2, 300, 64), _t(2, 8, 5, 64))


@pytest.mark.parametrize("op", ["flash_attn_mma_stages_split_q", "flash_attn_mma_stages_split_q_tiling_qk_swizzle_qkv",
                                "flash_attn_cute", "fmha_host"])
def test_reference_ops_stay_fp16(op):
    x = _t(1, 2, 64, 64)
    fn = getattr(flash_attn, op)
    with pytest.raises(RuntimeError, match="values must be torch::kHalf"):
        fn(x, x, x, x) if op in ("flash_attn_cute", "fmha_host") else fn(x, x, x, x, 1)


@pytest.mark.parametrize("op", ["ffpa_mma_acc_f32_L1", "ffpa_mma_acc_f16_L1"])
def test_ffpa_stays_fp16(op):
    from leetcuda_b200 import ffpa_attn
    x = _t(1, 2, 64, 320)
    with pytest.raises(RuntimeError, match="values must be torch::kHalf"):
        getattr(ffpa_attn, op)(x, x, x, x, 1)
