"""Argument checks of the fp8-K/V attention entries and of flash_attn.fmha_fwd with float8_e4m3fn K and V: rejected on
the host, before any CUDA call (no GPU needed).  The C entries b200_fmha_fwd_{f16,bf16}_fp8kv_seqlens / _paged run
exactly the checks, and give exactly the messages, of their counterparts (the argument tables of test_attn_seqlens_args
/ test_attn_paged_args are replayed against them), then their own: D % 16 and the two scales."""
import math

import pytest
import torch

import test_attn_paged_args as PA
import test_attn_seqlens_args as SA
from leetcuda_b200 import _capi, flash_attn

TYPES = ["f16", "bf16"]


def _table(test):
    return [m for m in test.pytestmark if m.name == "parametrize"][0].args[1]


class _Fp8Entries:
    """The f16 module's lib with its f16 entries answered by the fp8-K/V ones of Q/O type T at the given scales."""

    def __init__(self, lib, T, k_scale=1.0, v_scale=1.0):
        sl, pg = getattr(lib, f"b200_fmha_fwd_{T}_fp8kv_seqlens"), getattr(lib, f"b200_fmha_fwd_{T}_fp8kv_paged")
        self.b200_fmha_fwd_f16_seqlens = lambda *a: sl(*a[:-1], k_scale, v_scale, a[-1])
        self.b200_fmha_fwd_f16_paged = lambda *a: pg(*a[:-1], k_scale, v_scale, a[-1])


@pytest.mark.parametrize("T", TYPES)
@pytest.mark.parametrize("kw,text", _table(SA.test_c_argument_checks))
def test_c_seqlens_checks_match_counterpart(built_lib, kw, text, T):
    assert SA._sl(_Fp8Entries(built_lib, T), **kw) == SA._sl(built_lib, **kw) == -1
    ref = _capi.last_error()
    SA._sl(_Fp8Entries(built_lib, T), **kw)
    assert _capi.last_error() == ref and ref.startswith("fmha_seqlens: ") and text in ref


@pytest.mark.parametrize("T", TYPES)
@pytest.mark.parametrize("kw,text", _table(PA.test_c_argument_checks))
def test_c_paged_checks_match_counterpart(built_lib, kw, text, T):
    assert PA._pg(_Fp8Entries(built_lib, T), **kw) == PA._pg(built_lib, **kw) == -1
    ref = _capi.last_error()
    PA._pg(_Fp8Entries(built_lib, T), **kw)
    assert _capi.last_error() == ref and ref.startswith("fmha_paged: ") and text in ref


@pytest.mark.parametrize("T", TYPES)
@pytest.mark.parametrize("D", [100, 1032])
def test_c_head_dim_of_the_counterpart_first(built_lib, T, D):
    assert SA._sl(_Fp8Entries(built_lib, T), D=D, splits=0) == -3
    assert _capi.last_error().startswith("fmha_seqlens: headdim not support!")
    assert PA._pg(_Fp8Entries(built_lib, T), D=D, splits=0) == -3
    assert _capi.last_error().startswith("fmha_paged: headdim not support!")


@pytest.mark.parametrize("T", TYPES)
@pytest.mark.parametrize("D", [8, 24, 72, 136, 264, 1016])
def test_c_head_dim_multiple_of_16(built_lib, T, D):
    for call, who in ((SA._sl, "fmha_seqlens"), (PA._pg, "fmha_paged")):
        assert call(_Fp8Entries(built_lib, T), D=D) == -1
        err = _capi.last_error()
        assert err.startswith(f"{who}: fp8 K/V need D % 16 == 0") and f"got D={D}" in err, err


@pytest.mark.parametrize("T", TYPES)
@pytest.mark.parametrize("which", ["k_scale", "v_scale"])
@pytest.mark.parametrize("value", [0.0, -0.0, -1.0, math.nan, math.inf, -math.inf])
def test_c_scales_finite_and_positive(built_lib, T, which, value):
    scales = dict(k_scale=1.0, v_scale=1.0)
    scales[which] = value
    for call, who in ((SA._sl, "fmha_seqlens"), (PA._pg, "fmha_paged")):
        assert call(_Fp8Entries(built_lib, T, **scales)) == -1
        err = _capi.last_error()
        assert err.startswith(f"{who}: {which}=") and err.endswith("must be finite and > 0"), err


@pytest.mark.parametrize("T", TYPES)
def test_c_folded_scale_finite(built_lib, T):
    """scale = 1e4 and k_scale = 3e38 are each finite, their fp32 product is not."""
    for pre, who in (("seqlens", "fmha_seqlens"), ("paged", "fmha_paged")):
        fn = getattr(built_lib, f"b200_fmha_fwd_{T}_fp8kv_{pre}")
        args = ([16, 16, 16, 16, None, None, None, 2, 8, 2, 1, 128, 64, 0, 1, 1e4, 3e38, 1.0, None] if pre == "seqlens"
                else [16, 16, 16, 16, None, 16, None, None, 2, 8, 2, 1, 64, 16, 32, 64, 0, 1, 1e4, 3e38, 1.0, None])
        assert fn(*args) == -1
        assert _capi.last_error().startswith(f"{who}: scale*k_scale = inf must be finite and > 0")


# ------------------------------------------------------------------ Python
def _t(*shape, dtype=torch.bfloat16):
    return torch.zeros(*shape, dtype=dtype)


E4 = torch.float8_e4m3fn
E5 = torch.float8_e5m2
_DT = {"fp16": torch.float16, "bf16": torch.bfloat16, "fp32": torch.float32, "e4m3": E4, "e5m2": E5}
_KV = {False: (2, 2, 300, 64), True: (40, 16, 2, 64)}


def _call(dts, paged, **kw):
    q, k, v, o = (_DT[d] for d in dts.split())
    if paged:
        kw["block_table"] = torch.zeros(2, 8, dtype=torch.int32)
    flash_attn.fmha_fwd(_t(2, 8, 5, 64, dtype=q), _t(*_KV[paged], dtype=k), _t(*_KV[paged], dtype=v),
                        _t(2, 8, 5, 64, dtype=o), **kw)


@pytest.mark.parametrize("paged", [False, True], ids=["contiguous", "paged"])
@pytest.mark.parametrize("dts,text", [
    ("e4m3 e4m3 e4m3 bf16", "Q and O must be fp16 or bf16"), ("bf16 e4m3 e4m3 e4m3", "Q and O must be fp16 or bf16"),
    ("e4m3 bf16 bf16 bf16", "Q and O must be fp16 or bf16"),
    ("bf16 e5m2 e5m2 bf16", "must be float8_e4m3fn"), ("fp16 e4m3 e5m2 fp16", "must be float8_e4m3fn"),
    ("e5m2 fp16 fp16 fp16", "must be float8_e4m3fn"),
    ("bf16 e4m3 bf16 bf16", "K and V must share one dtype"), ("fp16 fp16 e4m3 fp16", "K and V must share one dtype"),
    ("bf16 e4m3 e4m3 fp16", "Q and O must both be fp16 or both bf16"),
    ("fp16 e4m3 e4m3 bf16", "Q and O must both be fp16 or both bf16"),
    ("fp32 e4m3 e4m3 fp32", "Q and O must both be fp16 or both bf16"),
])
def test_python_rejects_dtypes(dts, text, paged):
    with pytest.raises(RuntimeError, match=text):
        _call(dts, paged)


@pytest.mark.parametrize("extra", [{}, dict(seqlens_k=torch.zeros(2, dtype=torch.int32)),
                                   dict(block_table=torch.zeros(2, 8, dtype=torch.int32))],
                         ids=["dense", "seqlens", "paged"])
def test_python_rejects_transposed_v(extra):
    k = _t(40, 16, 2, 64, dtype=E4) if "block_table" in extra else _t(2, 2, 300, 64, dtype=E4)
    with pytest.raises(RuntimeError, match="transposed V is not supported with fp8 K/V"):
        flash_attn.fmha_fwd(_t(2, 8, 5, 64), k, _t(2, 2, 64, 300, dtype=E4), _t(2, 8, 5, 64), v_transposed=True,
                            **extra)


@pytest.mark.parametrize("dts", ["fp16 fp16 fp16 fp16", "bf16 bf16 bf16 bf16"])
@pytest.mark.parametrize("scales", [dict(k_scale=2.0), dict(v_scale=0.5), dict(k_scale=0.0, v_scale=3.0)])
@pytest.mark.parametrize("paged", [False, True], ids=["contiguous", "paged"])
def test_python_rejects_scales_without_fp8(dts, scales, paged):
    with pytest.raises(RuntimeError, match="k_scale / v_scale apply to fp8"):
        _call(dts, paged, **scales)


@pytest.mark.parametrize("dts", ["fp16 e4m3 e4m3 fp16", "bf16 e4m3 e4m3 bf16"])
def test_python_fp8_keeps_the_other_checks(dts):
    q, k, v, o = (_DT[d] for d in dts.split())
    with pytest.raises(RuntimeError, match="Tensor size mismatch!"):
        flash_attn.fmha_fwd(_t(2, 8, 5, 64, dtype=q), _t(2, 2, 300, 64, dtype=k), _t(2, 2, 300, 64, dtype=v),
                            _t(2, 8, 6, 64, dtype=o))
    with pytest.raises(RuntimeError, match="num_splits must be an int"):
        _call(dts, False, num_splits=65)
    with pytest.raises(RuntimeError, match=r"lse must be .*\[B,H,Nq\]"):
        _call(dts, False, lse=torch.zeros(2, 8, 6))
    with pytest.raises(RuntimeError, match="page_size .* must be a power of two"):
        flash_attn.fmha_fwd(_t(2, 8, 5, 64, dtype=q), _t(40, 24, 2, 64, dtype=k), _t(40, 24, 2, 64, dtype=v),
                            _t(2, 8, 5, 64, dtype=o), block_table=torch.zeros(2, 8, dtype=torch.int32))
    with pytest.raises(RuntimeError, match="tensors must be CUDA tensors"):
        _call(dts, False, k_scale=0.5, v_scale=2.0)
    with pytest.raises(RuntimeError, match="block_table must be an int32 contiguous CUDA tensor"):
        _call(dts, True, k_scale=0.5, v_scale=2.0)


@pytest.mark.parametrize("op", ["flash_attn_mma_stages_split_q", "flash_attn_cute", "fmha_host"])
def test_reference_ops_stay_fp16(op):
    x, k = _t(1, 2, 64, 64, dtype=torch.float16), _t(1, 2, 64, 64, dtype=E4)
    fn = getattr(flash_attn, op)
    with pytest.raises(RuntimeError, match="values must be torch::kHalf"):
        fn(x, k, k, x) if op in ("flash_attn_cute", "fmha_host") else fn(x, k, k, x, 1)
