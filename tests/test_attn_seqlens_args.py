"""Argument checks of b200_fmha_fwd_f16_seqlens and of flash_attn.fmha_fwd with seqlens_q / seqlens_k: rejected on the
host, before any CUDA call (no GPU needed)."""
import pytest
import torch

from leetcuda_b200 import _capi, flash_attn


def _sl(lib, q=16, k=16, v=16, o=16, sq=None, sk=None, B=2, H=8, Hkv=2, Nq=1, Nk=128, D=64, causal=0, splits=1):
    return lib.b200_fmha_fwd_f16_seqlens(q, k, v, o, None, sq, sk, B, H, Hkv, Nq, Nk, D, causal, splits, 0.0, None)


@pytest.mark.parametrize("kw,text", [
    (dict(q=None), "null pointer"), (dict(k=None), "null pointer"), (dict(v=None), "null pointer"),
    (dict(o=None), "null pointer"),
    (dict(B=0), "bad shape B=0"), (dict(H=-1), "bad shape"), (dict(D=0), "bad shape"),
    (dict(Nq=0), "bad lengths Nq=0 Nk=128"), (dict(Nk=-4), "bad lengths Nq=1 Nk=-4"),
    (dict(causal=2), "causal must be 0 or 1, got 2"), (dict(causal=-1), "causal must be 0 or 1, got -1"),
    (dict(Hkv=3), "Hkv=3 must be >= 1 and divide H=8"), (dict(Hkv=0), "Hkv=0 must be >= 1"),
    (dict(splits=-1), "num_splits=-1 must be in 0 .. 64"), (dict(splits=65), "num_splits=65 must be in 0 .. 64"),
    (dict(B=2, H=40000, Hkv=40000), "B*Hkv = 80000 exceeds the grid limit 65535"),
    (dict(o=18, splits=2), "o must be 16-byte aligned"), (dict(o=18, splits=0), "o must be 16-byte aligned"),
    (dict(H=65536, Hkv=1, Nq=2 ** 16), "(H/Hkv)*Nq = 4294967296 query rows per K/V head exceed 2^31 - 1"),
    (dict(sq=18), "seqlens_q must be 4-byte aligned"), (dict(sk=6), "seqlens_k must be 4-byte aligned"),
])
def test_c_argument_checks(built_lib, kw, text):
    assert _sl(built_lib, **kw) == -1
    err = _capi.last_error()
    assert err.startswith("fmha_seqlens: ") and text in err, err


@pytest.mark.parametrize("D", [100, 1032])
def test_c_head_dim(built_lib, D):
    assert _sl(built_lib, D=D, splits=0) == -3
    assert _capi.last_error().startswith("fmha_seqlens: headdim not support!")


def _t(*shape, dtype=torch.float16):
    return torch.zeros(*shape, dtype=dtype)


def _fwd(**kw):
    q, kv, o = _t(2, 8, 5, 64), _t(2, 2, 300, 64), _t(2, 8, 5, 64)
    flash_attn.fmha_fwd(q, kw.pop("k", kv), kw.pop("v", kv), o, **kw)


@pytest.mark.parametrize("name", ["seqlens_q", "seqlens_k"])
@pytest.mark.parametrize("value", [
    torch.zeros(2, dtype=torch.int64), torch.zeros(2, dtype=torch.float32), torch.zeros(3, dtype=torch.int32),
    torch.zeros(2, 1, dtype=torch.int32), torch.zeros(4, dtype=torch.int32)[::2], torch.zeros(2, dtype=torch.int32),
    [1, 2], 5,
], ids=["int64", "float32", "len3", "2x1", "strided", "cpu", "list", "int"])
def test_python_length_errors(name, value):
    with pytest.raises(RuntimeError, match=name + " must be an int32 contiguous CUDA tensor"):
        _fwd(**{name: value})


def test_python_transposed_v_with_lengths():
    for kw in (dict(seqlens_q=torch.zeros(2, dtype=torch.int32)), dict(seqlens_k=torch.zeros(2, dtype=torch.int32))):
        with pytest.raises(RuntimeError, match="v_transposed=True is not supported with lengths"):
            _fwd(v=_t(2, 2, 64, 300), v_transposed=True, **kw)


def test_python_shape_split_and_lse_errors():
    lens = dict(seqlens_k=torch.zeros(2, dtype=torch.int32))
    with pytest.raises(RuntimeError, match="Tensor size mismatch!"):
        _fwd(k=_t(2, 3, 300, 64), **lens)
    with pytest.raises(RuntimeError, match="num_splits must be an int"):
        _fwd(num_splits=65, **lens)
    with pytest.raises(RuntimeError, match=r"lse must be .*\[B,H,Nq\]"):
        _fwd(lse=torch.zeros(2, 8, 300), **lens)
