"""Argument checks of b200_fmha_fwd_f16_paged and of flash_attn.fmha_fwd with block_table: rejected on the host,
before any CUDA call (no GPU needed)."""
import pytest
import torch

from leetcuda_b200 import _capi, flash_attn


def _pg(lib, q=16, k=16, v=16, o=16, lse=None, table=16, sq=None, sk=None, B=2, H=8, Hkv=2, Nq=1, num_pages=64,
        page_size=16, max_pages=32, D=64, causal=0, splits=1):
    return lib.b200_fmha_fwd_f16_paged(q, k, v, o, lse, table, sq, sk, B, H, Hkv, Nq, num_pages, page_size, max_pages,
                                       D, causal, splits, 0.0, None)


@pytest.mark.parametrize("kw,text", [
    (dict(q=None), "null pointer"), (dict(k=None), "null pointer"), (dict(v=None), "null pointer"),
    (dict(o=None), "null pointer"), (dict(table=None), "null pointer (q, k_cache, v_cache, o and block_table"),
    (dict(B=0), "bad shape B=0"), (dict(H=-1), "bad shape"), (dict(D=0), "bad shape"),
    (dict(Nq=0), "bad length Nq=0"),
    (dict(causal=2), "causal must be 0 or 1, got 2"), (dict(causal=-1), "causal must be 0 or 1, got -1"),
    (dict(Hkv=3), "Hkv=3 must be >= 1 and divide H=8"), (dict(Hkv=0), "Hkv=0 must be >= 1"),
    (dict(splits=-1), "num_splits=-1 must be in 0 .. 64"), (dict(splits=65), "num_splits=65 must be in 0 .. 64"),
    (dict(B=2, H=40000, Hkv=40000), "B*Hkv = 80000 exceeds the grid limit 65535"),
    (dict(o=18, splits=2), "o must be 16-byte aligned"), (dict(o=18, splits=0), "o must be 16-byte aligned"),
    (dict(H=65536, Hkv=1, Nq=2 ** 16), "(H/Hkv)*Nq = 4294967296 query rows per K/V head exceed 2^31 - 1"),
    (dict(sq=18), "seqlens_q must be 4-byte aligned"), (dict(sk=6), "seqlens_k must be 4-byte aligned"),
    (dict(table=18), "block_table must be 4-byte aligned"),
    (dict(num_pages=0), "num_pages=0 must be >= 1"), (dict(max_pages=0), "max_pages_per_seq=0 must be >= 1"),
    (dict(page_size=8), "page_size=8 must be a power of two >= 16"),
    (dict(page_size=48), "page_size=48 must be a power of two >= 16"),
    (dict(page_size=0), "page_size=0 must be a power of two >= 16"),
    (dict(num_pages=2 ** 27), "num_pages*page_size = 2147483648 pool rows exceed 2^31 - 1"),
    (dict(max_pages=2 ** 27), "max_pages_per_seq*page_size = 2147483648 keys per sequence exceed 2^31 - 1"),
])
def test_c_argument_checks(built_lib, kw, text):
    assert _pg(built_lib, **kw) == -1
    err = _capi.last_error()
    assert err.startswith("fmha_paged: ") and text in err, err


@pytest.mark.parametrize("D", [100, 1032])
def test_c_head_dim(built_lib, D):
    assert _pg(built_lib, D=D, splits=0) == -3
    assert _capi.last_error().startswith("fmha_paged: headdim not support!")


def _t(*shape, dtype=torch.float16):
    return torch.zeros(*shape, dtype=dtype)


def _fwd(**kw):
    q, pool, o = _t(2, 8, 5, 64), _t(40, 16, 2, 64), _t(2, 8, 5, 64)
    kw.setdefault("block_table", torch.zeros(2, 8, dtype=torch.int32))
    flash_attn.fmha_fwd(q, kw.pop("k", pool), kw.pop("v", pool), o, **kw)


@pytest.mark.parametrize("value", [
    torch.zeros(2, 8, dtype=torch.int64), torch.zeros(2, 8, dtype=torch.float32), torch.zeros(3, 8, dtype=torch.int32),
    torch.zeros(2, dtype=torch.int32), torch.zeros(2, 0, dtype=torch.int32), torch.zeros(2, 16, dtype=torch.int32)[:, ::2],
    torch.zeros(2, 8, dtype=torch.int32), [[0] * 8] * 2,
], ids=["int64", "float32", "3x8", "1d", "2x0", "strided", "cpu", "list"])
def test_python_block_table_errors(value):
    with pytest.raises(RuntimeError, match=r"block_table must be an int32 contiguous CUDA tensor \[B, max_pages_per_seq\]"):
        _fwd(block_table=value)


@pytest.mark.parametrize("k,v", [
    (_t(40, 16, 2, 32), _t(40, 16, 2, 32)),     # D differs from Q's
    (_t(40, 16, 3, 64), _t(40, 16, 3, 64)),     # Hkv does not divide H
    (_t(40, 16, 2, 64), _t(41, 16, 2, 64)),     # K and V pools differ
    (_t(40, 16, 2, 64), _t(40, 32, 2, 64)),
    (_t(2, 2, 300, 64), _t(2, 2, 300, 64)[0]),  # not 4-d
    (_t(0, 16, 2, 64), _t(0, 16, 2, 64)),       # no page
])
def test_python_pool_shape_errors(k, v):
    with pytest.raises(RuntimeError, match=r"K and V must be pools \[num_pages, page_size, Hkv, D\]"):
        _fwd(k=k, v=v)


@pytest.mark.parametrize("page_size", [8, 24, 1])
def test_python_page_size(page_size):
    pool = _t(40, page_size, 2, 64)
    with pytest.raises(RuntimeError, match=f"page_size \\(K.shape\\[1\\]\\) must be a power of two >= 16, got {page_size}"):
        _fwd(k=pool, v=pool)


def test_python_pool_dtype_and_transposed_v():
    pool = _t(40, 16, 2, 64, dtype=torch.float32)
    with pytest.raises(RuntimeError, match="values must be torch::kHalf"):
        _fwd(k=pool, v=pool)
    with pytest.raises(RuntimeError, match="v_transposed=True is not supported with a block table"):
        _fwd(v_transposed=True)


@pytest.mark.parametrize("name", ["seqlens_q", "seqlens_k"])
def test_python_length_errors(name):
    with pytest.raises(RuntimeError, match=name + " must be an int32 contiguous CUDA tensor"):
        _fwd(block_table=torch.zeros(2, 8, dtype=torch.int32), **{name: torch.zeros(3, dtype=torch.int32)})


def test_python_split_and_lse_errors():
    with pytest.raises(RuntimeError, match="num_splits must be an int"):
        _fwd(num_splits=65)
    with pytest.raises(RuntimeError, match=r"lse must be .*\[B,H,Nq\]"):
        _fwd(lse=torch.zeros(2, 8, 300))
    with pytest.raises(RuntimeError, match="Tensor size mismatch!"):
        q = _t(2, 8, 5, 64)
        flash_attn.fmha_fwd(q, _t(40, 16, 2, 64), _t(40, 16, 2, 64), _t(2, 8, 6, 64),
                            block_table=torch.zeros(2, 8, dtype=torch.int32))
