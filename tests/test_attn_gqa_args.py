"""Argument checks of b200_fmha_fwd_f16_gqa and of flash_attn.fmha_fwd with grouped K/V heads and num_splits: rejected
on the host, before any CUDA call (no GPU needed)."""
import pytest
import torch

from leetcuda_b200 import _capi, flash_attn


def _gqa(lib, B=1, H=8, Hkv=2, Nq=1, Nk=128, D=64, vt=0, causal=0, splits=1):
    return lib.b200_fmha_fwd_f16_gqa(16, 16, 16, 16, None, B, H, Hkv, Nq, Nk, D, vt, causal, splits, 0.0, None)


@pytest.mark.parametrize("H,Hkv", [(8, 0), (8, -2), (8, 3), (4, 8), (6, 4)])
def test_kv_heads_must_divide_query_heads(built_lib, H, Hkv):
    assert _gqa(built_lib, H=H, Hkv=Hkv) == -1
    assert f"Hkv={Hkv} must be >= 1 and divide H={H}" in _capi.last_error()


@pytest.mark.parametrize("splits", [-1, -7, _capi.FMHA_MAX_SPLITS + 1, 1000])
def test_num_splits_range(built_lib, splits):
    assert _gqa(built_lib, splits=splits) == -1
    assert f"num_splits={splits} must be in 0 .. {_capi.FMHA_MAX_SPLITS}" in _capi.last_error()


def test_grid_limit_is_on_kv_heads(built_lib):
    assert _gqa(built_lib, B=2, H=40000, Hkv=40000) == -1
    assert "B*Hkv = 80000 exceeds the grid limit 65535" in _capi.last_error()
    # B*H above the limit with B*Hkv below it passes this check: the next one (null pointers) is what fails
    rc = built_lib.b200_fmha_fwd_f16_gqa(None, 16, 16, 16, None, 2, 40000, 8, 1, 64, 64, 0, 0, 1, 0.0, None)
    assert rc == -1 and "null pointer" in _capi.last_error()


@pytest.mark.parametrize("Nq,Nk", [(0, 128), (128, 0), (-1, 128), (128, -5)])
def test_lengths_must_be_positive(built_lib, Nq, Nk):
    assert _gqa(built_lib, Nq=Nq, Nk=Nk) == -1
    assert f"Nq={Nq} Nk={Nk}" in _capi.last_error()


@pytest.mark.parametrize("causal", [-1, 2])
def test_causal_is_a_flag(built_lib, causal):
    assert _gqa(built_lib, causal=causal) == -1
    assert "causal must be 0 or 1" in _capi.last_error()


def test_transposed_v_needs_nk_multiple_of_8(built_lib):
    assert _gqa(built_lib, Nq=64, Nk=100, vt=1) == -1
    assert "Nk (100) must be a multiple of 8" in _capi.last_error()


@pytest.mark.parametrize("D,code", [(100, -3), (1032, -3), (0, -1)])
def test_head_dim(built_lib, D, code):
    assert _gqa(built_lib, D=D, splits=0) == code
    assert ("headdim not support" if code == -3 else "bad shape") in _capi.last_error()


def test_null_pointer_and_batch(built_lib):
    rc = built_lib.b200_fmha_fwd_f16_gqa(16, None, 16, 16, None, 1, 8, 2, 1, 64, 64, 0, 0, 0, 0.0, None)
    assert rc == -1 and "null pointer" in _capi.last_error()
    assert _gqa(built_lib, B=0) == -1 and "bad shape" in _capi.last_error()


def _t(*shape):
    return torch.zeros(*shape, dtype=torch.float16)


@pytest.mark.parametrize("k_shape,v_shape,o_shape", [
    ((2, 3, 300, 64), (2, 3, 300, 64), (2, 8, 100, 64)),    # K heads do not divide H
    ((2, 16, 300, 64), (2, 16, 300, 64), (2, 8, 100, 64)),  # more K heads than Q heads
    ((2, 2, 300, 64), (2, 4, 300, 64), (2, 8, 100, 64)),    # V heads != K heads
    ((2, 4, 300, 64), (2, 2, 300, 64), (2, 8, 100, 64)),    # V heads != K heads
    ((2, 2, 300, 64), (2, 2, 300, 64), (2, 2, 100, 64)),    # O follows Q, not K
    ((2, 2, 300, 64), (2, 2, 299, 64), (2, 8, 100, 64)),    # V length != K length
    ((1, 2, 300, 64), (1, 2, 300, 64), (2, 8, 100, 64)),    # K batch
])
def test_fmha_fwd_shape_errors(k_shape, v_shape, o_shape):
    with pytest.raises(RuntimeError, match="Tensor size mismatch!"):
        flash_attn.fmha_fwd(_t(2, 8, 100, 64), _t(*k_shape), _t(*v_shape), _t(*o_shape), causal=True, num_splits=0)


def test_fmha_fwd_grouped_transposed_v():
    q, k = _t(2, 8, 100, 64), _t(2, 2, 304, 64)
    with pytest.raises(RuntimeError, match="Tensor size mismatch!"):
        flash_attn.fmha_fwd(q, k, _t(2, 8, 64, 304), _t(2, 8, 100, 64), v_transposed=True)
    with pytest.raises(RuntimeError, match="no CPU path"):   # the right layout passes the shape check
        flash_attn.fmha_fwd(q, k, _t(2, 2, 64, 304), _t(2, 8, 100, 64), v_transposed=True)


def test_fmha_fwd_lse_follows_q():
    q, kv = _t(2, 8, 100, 64), _t(2, 2, 300, 64)
    for shape in [(2, 2, 100), (2, 8, 300), (2, 8, 100, 1)]:
        with pytest.raises(RuntimeError, match=r"lse must be .*\[B,H,Nq\]"):
            flash_attn.fmha_fwd(q, kv, kv, _t(2, 8, 100, 64), lse=torch.zeros(shape), num_splits=2)
    with pytest.raises(RuntimeError, match="no CPU path"):
        flash_attn.fmha_fwd(q, kv, kv, _t(2, 8, 100, 64), lse=torch.zeros(2, 8, 100), num_splits=2)


@pytest.mark.parametrize("splits", [-1, _capi.FMHA_MAX_SPLITS + 1, 2.0, "2", None, True])
def test_fmha_fwd_bad_num_splits(splits):
    q, kv = _t(1, 4, 1, 64), _t(1, 2, 300, 64)
    with pytest.raises(RuntimeError, match="num_splits must be an int"):
        flash_attn.fmha_fwd(q, kv, kv, _t(1, 4, 1, 64), num_splits=splits)


def test_reference_ops_keep_all_heads():
    """The reference op names and flash_attn_cute still demand K and V with Q's head count."""
    q, kv = _t(1, 4, 128, 64), _t(1, 2, 128, 64)
    with pytest.raises(RuntimeError, match="Tensor size mismatch!"):
        flash_attn.flash_attn_mma_stages_split_q_shared_qkv(q, kv, kv, _t(1, 4, 128, 64), 1)
    with pytest.raises(RuntimeError, match="Tensor size mismatch!"):
        flash_attn.flash_attn_cute(q, kv, kv, _t(1, 4, 128, 64))


def test_split_output_must_be_16_byte_aligned(built_lib):
    """The combine stores 16-byte packs of O: with num_splits != 1 a misaligned o is rejected, with 1 it passes this
    check (the null k is what fails then)."""
    for splits in (0, 2):
        rc = built_lib.b200_fmha_fwd_f16_gqa(16, 16, 16, 18, None, 1, 8, 2, 1, 128, 64, 0, 0, splits, 0.0, None)
        assert rc == -1 and "o must be 16-byte aligned" in _capi.last_error()
    rc = built_lib.b200_fmha_fwd_f16_gqa(16, None, 16, 18, None, 1, 8, 2, 1, 128, 64, 0, 0, 1, 0.0, None)
    assert rc == -1 and "null pointer" in _capi.last_error()


@pytest.mark.parametrize("args,text", [
    ((0, 8, 2, 1, 128, 64), "bad shape"), ((1, 8, 3, 1, 128, 64), "Hkv=3 must be >= 1 and divide H=8"),
    ((1, 8, 2, 0, 128, 64), "bad shape"), ((1, 8, 0, 1, 128, 64), "Hkv=0"),
])
def test_split_count_query_arguments(built_lib, args, text):
    assert built_lib.b200_fmha_fwd_f16_gqa_splits(*args) == -1
    assert text in _capi.last_error()
