"""Argument checks of b200_fmha_fwd_f16_kv and of flash_attn.fmha_fwd with separate query / key lengths: rejected on
the host, before any CUDA call (no GPU needed)."""
import pytest
import torch

from leetcuda_b200 import flash_attn


def _kv(lib, B=1, H=1, Nq=128, Nk=128, D=64, vt=0, causal=0):
    return lib.b200_fmha_fwd_f16_kv(16, 16, 16, 16, None, B, H, Nq, Nk, D, vt, causal, 0.0, None)


@pytest.mark.parametrize("Nq,Nk", [(0, 128), (128, 0), (-1, 128), (128, -5)])
def test_lengths_must_be_positive(built_lib, Nq, Nk):
    from leetcuda_b200 import _capi
    assert _kv(built_lib, Nq=Nq, Nk=Nk) == -1
    assert f"Nq={Nq} Nk={Nk}" in _capi.last_error()


@pytest.mark.parametrize("causal", [-1, 2, 7])
def test_causal_is_a_flag(built_lib, causal):
    from leetcuda_b200 import _capi
    assert _kv(built_lib, causal=causal) == -1
    assert "causal must be 0 or 1" in _capi.last_error()


def test_transposed_v_needs_nk_multiple_of_8(built_lib):
    from leetcuda_b200 import _capi
    assert _kv(built_lib, Nq=64, Nk=100, vt=1) == -1
    assert "Nk (100) must be a multiple of 8" in _capi.last_error()


def test_head_dim_multiple_of_8(built_lib):
    from leetcuda_b200 import _capi
    assert _kv(built_lib, Nq=1, Nk=777, D=100, causal=1) == -3
    assert "headdim not support" in _capi.last_error()


def test_grid_limit(built_lib):
    from leetcuda_b200 import _capi
    assert _kv(built_lib, B=2, H=40000, Nq=1, Nk=64, causal=1) == -1
    assert "grid limit" in _capi.last_error()


def _t(*shape):
    return torch.zeros(*shape, dtype=torch.float16)


@pytest.mark.parametrize("k_shape,v_shape,o_shape", [
    ((2, 4, 300, 64), (2, 4, 300, 64), (1, 4, 100, 64)),    # O batch
    ((2, 3, 300, 64), (2, 3, 300, 64), (2, 4, 100, 64)),    # K heads
    ((2, 4, 300, 32), (2, 4, 300, 64), (2, 4, 100, 64)),    # K head dim
    ((2, 4, 300, 64), (2, 4, 299, 64), (2, 4, 100, 64)),    # V length != K length
    ((2, 4, 300, 64), (2, 4, 64, 300), (2, 4, 100, 64)),    # V transposed although v_transposed=False
    ((2, 4, 300, 64), (2, 4, 300, 64), (2, 4, 300, 64)),    # O follows Q, not K
])
def test_fmha_fwd_shape_errors(k_shape, v_shape, o_shape):
    with pytest.raises(RuntimeError, match="Tensor size mismatch!"):
        flash_attn.fmha_fwd(_t(2, 4, 100, 64), _t(*k_shape), _t(*v_shape), _t(*o_shape), causal=True)


def test_fmha_fwd_transposed_v_shape_error():
    q, k = _t(2, 4, 100, 64), _t(2, 4, 304, 64)
    with pytest.raises(RuntimeError, match="Tensor size mismatch!"):
        flash_attn.fmha_fwd(q, k, _t(2, 4, 304, 64), _t(2, 4, 100, 64), v_transposed=True)
    with pytest.raises(RuntimeError, match="no CPU path"):   # the right layout passes the shape check
        flash_attn.fmha_fwd(q, k, _t(2, 4, 64, 304), _t(2, 4, 100, 64), v_transposed=True)


def test_fmha_fwd_lse_follows_q():
    q, kv = _t(2, 4, 100, 64), _t(2, 4, 300, 64)
    for shape in [(2, 4, 300), (2, 4, 100, 1), (2, 100)]:
        with pytest.raises(RuntimeError, match=r"lse must be .*\[B,H,Nq\]"):
            flash_attn.fmha_fwd(q, kv, kv, _t(2, 4, 100, 64), lse=torch.zeros(shape), causal=True)
    with pytest.raises(RuntimeError, match="no CPU path"):
        flash_attn.fmha_fwd(q, kv, kv, _t(2, 4, 100, 64), lse=torch.zeros(2, 4, 100), causal=True)


def test_reference_ops_keep_one_length():
    """The reference op names and flash_attn_cute still demand one sequence length."""
    q, kv = _t(1, 2, 128, 64), _t(1, 2, 256, 64)
    with pytest.raises(RuntimeError, match="Tensor size mismatch!"):
        flash_attn.flash_attn_mma_stages_split_q_shared_qkv(q, kv, kv, _t(1, 2, 128, 64), 1)
    with pytest.raises(RuntimeError, match="Tensor size mismatch!"):
        flash_attn.flash_attn_cute(q, kv, kv, _t(1, 2, 128, 64))
