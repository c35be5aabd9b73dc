"""Argument checks of b200_fmha_fwd_{f16,bf16}_varlen / _varlen_paged and of flash_attn.fmha_varlen_fwd: rejected on
the host with a message that names the argument, before any CUDA call (no GPU needed: no launch is counted)."""
import pytest
import torch

from leetcuda_b200 import _capi, flash_attn

ENTRIES = ["b200_fmha_fwd_f16_varlen", "b200_fmha_fwd_bf16_varlen"]
PAGED = ["b200_fmha_fwd_f16_varlen_paged", "b200_fmha_fwd_bf16_varlen_paged"]


def _vl(lib, entry, q=16, k=16, v=16, o=16, lse=None, cq=16, ck=16, B=2, H=8, Hkv=2, total_q=100, total_k=100,
        max_q=64, max_k=64, D=64, causal=0):
    return getattr(lib, entry)(q, k, v, o, lse, cq, ck, B, H, Hkv, total_q, total_k, max_q, max_k, D, causal, 0.0, None)


def _pg(lib, entry, q=16, k=16, v=16, o=16, lse=None, cq=16, used=16, table=16, B=2, H=8, Hkv=2, total_q=100, max_q=64,
        num_pages=64, page_size=16, max_pages=32, D=64, causal=0):
    return getattr(lib, entry)(q, k, v, o, lse, cq, used, table, B, H, Hkv, total_q, max_q, num_pages, page_size,
                               max_pages, D, causal, 0.0, None)


_COMMON = [
    (dict(q=None), "null pointer"), (dict(k=None), "null pointer"), (dict(v=None), "null pointer"),
    (dict(o=None), "null pointer"), (dict(cq=None), "null pointer"),
    (dict(B=0), "bad shape B=0"), (dict(H=-1), "bad shape"), (dict(D=0), "bad shape"),
    (dict(total_q=0), "total_q=0 must be >= 1"), (dict(max_q=0), "max_seqlen_q=0 must be >= 1"),
    (dict(causal=2), "causal must be 0 or 1, got 2"), (dict(causal=-1), "causal must be 0 or 1, got -1"),
    (dict(Hkv=3), "Hkv=3 must be >= 1 and divide H=8"), (dict(Hkv=0), "Hkv=0 must be >= 1"),
    (dict(B=2, H=40000, Hkv=40000), "B*Hkv = 80000 exceeds the grid limit 65535"),
    (dict(cq=18), "cu_seqlens_q must be 4-byte aligned"),
    (dict(H=65536, Hkv=1, max_q=2 ** 16), "(H/Hkv)*max_seqlen_q = 4294967296 query rows per K/V head exceed 2^31 - 1"),
    (dict(H=2 ** 30, Hkv=1, max_q=1, total_q=1, D=1024), "CTAs exceed the grid limit 2^31 - 1"),
    (dict(B=1, total_q=2 ** 31 - 1, H=2 ** 31 - 1, Hkv=1, D=1024),
     "total_q*H*D = 2147483647*2147483647*1024 elements overflow"),
]


@pytest.mark.parametrize("entry", ENTRIES)
@pytest.mark.parametrize("kw,text", _COMMON + [
    (dict(ck=None), "null pointer (q, k, v, o, cu_seqlens_q and cu_seqlens_k are required)"),
    (dict(total_k=0), "total_k=0 must be >= 1"), (dict(max_k=0), "max_seqlen_k=0 must be >= 1"),
    (dict(ck=6), "cu_seqlens_k must be 4-byte aligned"),
])
def test_c_argument_checks(built_lib, entry, kw, text):
    n0 = _capi.launch_count()
    assert _vl(built_lib, entry, **kw) == -1
    err = _capi.last_error()
    assert err.startswith("fmha_varlen: ") and text in err, err
    assert _capi.launch_count() == n0


@pytest.mark.parametrize("entry", PAGED)
@pytest.mark.parametrize("kw,text", _COMMON + [
    (dict(table=None), "null pointer (block_table is required)"),
    (dict(used=None), "null pointer (q, k_cache, v_cache, o, cu_seqlens_q, seqused_k and block_table are required)"),
    (dict(used=6), "seqused_k must be 4-byte aligned"), (dict(table=18), "block_table must be 4-byte aligned"),
    (dict(num_pages=0), "num_pages=0 must be >= 1"), (dict(max_pages=0), "max_pages_per_seq=0 must be >= 1"),
    (dict(page_size=8), "page_size=8 must be a power of two >= 16"),
    (dict(page_size=48), "page_size=48 must be a power of two >= 16"),
    (dict(num_pages=2 ** 27), "num_pages*page_size = 2147483648 pool rows exceed 2^31 - 1"),
    (dict(max_pages=2 ** 27), "max_pages_per_seq*page_size = 2147483648 keys per sequence exceed 2^31 - 1"),
])
def test_c_paged_argument_checks(built_lib, entry, kw, text):
    n0 = _capi.launch_count()
    assert _pg(built_lib, entry, **kw) == -1
    err = _capi.last_error()
    assert err.startswith("fmha_varlen_paged: ") and text in err, err
    assert _capi.launch_count() == n0


@pytest.mark.parametrize("entry", ENTRIES + PAGED)
@pytest.mark.parametrize("D", [100, 1032])
def test_c_head_dim(built_lib, entry, D):
    n0 = _capi.launch_count()
    assert (_pg if entry in PAGED else _vl)(built_lib, entry, D=D) == -3
    assert "headdim not support!" in _capi.last_error()
    assert _capi.launch_count() == n0


# ------------------------------------------------------------------ Python
def _t(*shape, dtype=torch.float16):
    return torch.zeros(*shape, dtype=dtype)


def _fwd(**kw):
    q, o = kw.pop("q", _t(100, 8, 64)), kw.pop("o", _t(100, 8, 64))
    k, v = kw.pop("k", _t(90, 2, 64)), kw.pop("v", _t(90, 2, 64))
    cq, ck = kw.pop("cu_seqlens_q", torch.zeros(3, dtype=torch.int32)), kw.pop("cu_seqlens_k", torch.zeros(3, dtype=torch.int32))
    flash_attn.fmha_varlen_fwd(q, k, v, o, cq, ck, kw.pop("max_seqlen_q", 64), kw.pop("max_seqlen_k", 64), **kw)


@pytest.mark.parametrize("kw,text", [
    (dict(num_splits=2), "num_splits=2 is not supported"), (dict(num_splits=0), "num_splits=0 is not supported"),
    (dict(v_transposed=True), "v_transposed=True is not supported"),
    (dict(rms_g=1.0), "the fused RMS norm (rms_g=1.0) is not supported"),
])
def test_python_unsupported_options(kw, text):
    with pytest.raises(RuntimeError, match=text.replace("(", r"\(").replace(")", r"\)")):
        _fwd(**kw)


def test_python_fp8_rejected():
    k8 = _t(90, 2, 64).to(torch.float8_e4m3fn)
    with pytest.raises(RuntimeError, match="fp8 K/V is not supported with varlen"):
        _fwd(k=k8, v=k8)


@pytest.mark.parametrize("kw", [
    dict(k=_t(90, 2, 64, dtype=torch.bfloat16), v=_t(90, 2, 64, dtype=torch.bfloat16)),
    dict(o=_t(100, 8, 64, dtype=torch.float32)),
    dict(q=_t(100, 8, 64, dtype=torch.float32), o=_t(100, 8, 64, dtype=torch.float32),
         k=_t(90, 2, 64, dtype=torch.float32), v=_t(90, 2, 64, dtype=torch.float32)),
], ids=["mixed", "fp32-o", "fp32"])
def test_python_dtype(kw):
    with pytest.raises(RuntimeError, match="q, k, v and o must share one dtype, fp16 or bf16"):
        _fwd(**kw)


@pytest.mark.parametrize("kw,text", [
    (dict(q=_t(2, 50, 8, 64)), r"q and o must be \[total_q, H, D\]"),
    (dict(o=_t(101, 8, 64)), r"q and o must be \[total_q, H, D\]"),
    (dict(k=_t(90, 3, 64), v=_t(90, 3, 64)), r"k and v must be \[total_k, Hkv, D\]"),
    (dict(k=_t(90, 2, 32), v=_t(90, 2, 32)), r"k and v must be \[total_k, Hkv, D\]"),
    (dict(v=_t(91, 2, 64)), r"k and v must be \[total_k, Hkv, D\]"),
    (dict(max_seqlen_q=64.0), "max_seqlen_q must be an int"), (dict(max_seqlen_k=True), "max_seqlen_k must be an int"),
    (dict(lse=_t(100, 8, dtype=torch.float32)), r"lse must be a contiguous fp32 CUDA tensor \[H, total_q\] = \[8, 100\]"),
    (dict(lse=_t(8, 100)), r"lse must be a contiguous fp32 CUDA tensor \[H, total_q\]"),
    (dict(cu_seqlens_q=torch.zeros(1, dtype=torch.int32)), r"cu_seqlens_q must be an int32 contiguous CUDA tensor \[B \+ 1\]"),
    (dict(cu_seqlens_q=None), r"cu_seqlens_q must be an int32 contiguous CUDA tensor \[B \+ 1\]"),
    (dict(cu_seqlens_q=torch.zeros(3, dtype=torch.int64)), r"cu_seqlens_q must be an int32 contiguous CUDA tensor \[3\]"),
    (dict(cu_seqlens_q=torch.zeros(3, dtype=torch.int32)), r"cu_seqlens_q must be an int32 contiguous CUDA tensor \[3\]"),
    (dict(cu_seqlens_k=torch.zeros(4, dtype=torch.int32)), r"cu_seqlens_k must be an int32 contiguous CUDA tensor \[3\]"),
    (dict(cu_seqlens_k=None), r"cu_seqlens_k must be an int32 contiguous CUDA tensor \[3\]"),
    (dict(seqused_k=torch.zeros(2, dtype=torch.int32)), "seqused_k needs block_table"),
], ids=lambda x: None if isinstance(x, dict) else x[:30])
def test_python_argument_errors(kw, text):
    with pytest.raises(RuntimeError, match=text):
        _fwd(**kw)


def _paged(**kw):
    pool = kw.pop("pool", _t(40, 16, 2, 64))
    kw.setdefault("block_table", torch.zeros(2, 8, dtype=torch.int32))
    kw.setdefault("seqused_k", torch.zeros(2, dtype=torch.int32))
    kw.setdefault("cu_seqlens_k", None)
    _fwd(k=kw.pop("k", pool), v=kw.pop("v", pool), **kw)


@pytest.mark.parametrize("kw,text", [
    (dict(cu_seqlens_k=torch.zeros(3, dtype=torch.int32)), "with block_table, cu_seqlens_k must be None"),
    (dict(pool=_t(40, 16, 3, 64)), r"k and v must be pools \[num_pages, page_size, Hkv, D\]"),
    (dict(pool=_t(0, 16, 2, 64)), r"k and v must be pools \[num_pages, page_size, Hkv, D\]"),
    (dict(k=_t(40, 16, 2, 64), v=_t(41, 16, 2, 64)), r"k and v must be pools \[num_pages, page_size, Hkv, D\]"),
    (dict(pool=_t(40, 24, 2, 64)), r"page_size \(k.shape\[1\]\) must be a power of two >= 16, got 24"),
    (dict(block_table=torch.zeros(3, 8, dtype=torch.int32)), r"block_table must be an int32 contiguous CUDA tensor"),
    (dict(block_table=torch.zeros(2, 8, dtype=torch.int64)), r"block_table must be an int32 contiguous CUDA tensor"),
    (dict(block_table=torch.zeros(2, 8, dtype=torch.int32)), r"block_table must be an int32 contiguous CUDA tensor"),
    (dict(block_table=torch.zeros(2, 16, dtype=torch.int32)[:, ::2]), r"block_table must be an int32 contiguous"),
], ids=lambda x: None if isinstance(x, dict) else x[:30])
def test_python_paged_errors(kw, text):
    with pytest.raises(RuntimeError, match=text):
        _paged(**kw)


def test_python_name_is_not_a_reference_op():
    assert "fmha_varlen_fwd" not in flash_attn.OP_NAMES
    assert "fmha_varlen_fwd" in flash_attn.__all__
