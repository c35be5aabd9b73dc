"""Argument checks of the KV-cache append: the C entries b200_kvcache_append_{f16,bf16}[_paged] and the Python
functions flash_attn.kvcache_append / fmha_fwd_kvcache reject every bad argument on the host, with a message naming it,
before any CUDA call and without a launch (_capi.launch_count() unchanged).  No GPU needed: the pointers are fake
addresses that are never dereferenced."""
import math
import re

import pytest
import torch

from leetcuda_b200 import _capi, flash_attn

# fake, 16-byte aligned, disjoint device addresses (the checks never dereference them)
A = {n: (i + 1) << 32 for i, n in enumerate(["k_new", "v_new", "k_cache", "v_cache", "block_table", "cache_seqlens",
                                                "seqlens_out", "q", "q_out", "cos", "sin"])}
GOOD = dict(B=2, H=8, Hkv=2, n_new=4, Nk=64, num_pages=10, page_size=16, max_pages_per_seq=4, D=64, rotary_dim=64,
            rotary_len=68, rotary_interleaved=0, cache_dtype=1, k_scale=1.0, v_scale=1.0)


def _call(lib, T="f16", paged=False, **kw):
    a = dict(A, **GOOD)
    a.update(kw)
    ptrs = [a["k_new"], a["v_new"], a["k_cache"], a["v_cache"]]
    tail = [a["D"], a["rotary_dim"], a["rotary_len"], a["rotary_interleaved"], a["cache_dtype"], a["k_scale"],
            a["v_scale"], None]
    mid = [a["cache_seqlens"], a["seqlens_out"], a["q"], a["q_out"], a["cos"], a["sin"], a["B"], a["H"], a["Hkv"],
           a["n_new"]]
    if paged:
        args = ptrs + [a["block_table"]] + mid + [a["num_pages"], a["page_size"], a["max_pages_per_seq"]] + tail
        fn = getattr(lib, f"b200_kvcache_append_{T}_paged")
    else:
        args = ptrs + mid + [a["Nk"]] + tail
        fn = getattr(lib, f"b200_kvcache_append_{T}")
    n0 = _capi.launch_count()
    rc = fn(*args)
    assert _capi.launch_count() == n0
    return rc


BAD = [
    (dict(k_new=None), "k_new is NULL"), (dict(v_cache=None), "v_cache is NULL"),
    (dict(cache_seqlens=None), "cache_seqlens is NULL"),
    (dict(q_out=None), "q and q_out must both be NULL or both be set"),
    (dict(sin=None), "rotary_cos and rotary_sin must both be NULL or both be set"),
    (dict(B=0), "B=0 must be >= 1"), (dict(H=0), "H=0 must be >= 1"), (dict(Hkv=0), "Hkv=0 must be >= 1"),
    (dict(n_new=0), "n_new=0 must be >= 1"), (dict(D=0), "D=0 must be >= 1"),
    (dict(H=6, Hkv=4), "Hkv=4 must divide H=6"),
    (dict(cache_dtype=2), "cache_dtype=2 must be 1"), (dict(cache_dtype=0), "cache_dtype=0 must be 1"),
    (dict(D=60, rotary_dim=48), "D=60 must be a multiple of 8"),
    (dict(D=72, rotary_dim=64, cache_dtype=3), "D=72 must be a multiple of 16 with an e4m3 cache"),
    (dict(rotary_dim=24), "rotary_dim=24 must be a multiple of 16"),
    (dict(rotary_dim=80), "rotary_dim=80 must be a multiple of 16 in 16 .. D=64"),
    (dict(rotary_dim=0), "rotary_dim=0 must be a multiple of 16"),
    (dict(rotary_interleaved=2), "rotary_interleaved must be 0 or 1"),
    (dict(cos=None, sin=None), "rotary_dim, rotary_len and rotary_interleaved must be 0 without rotary tables"),
    (dict(k_scale=2.0), "k_scale=2 must be 1 unless the cache is e4m3"),
    (dict(v_scale=0.5), "v_scale=0.5 must be 1 unless the cache is e4m3"),
    (dict(k_new=A["k_new"] + 8), "k_new must be 16-byte aligned"),
    (dict(q_out=A["q_out"] + 4), "q_out must be 16-byte aligned"),
    (dict(cos=A["cos"] + 4), "rotary_cos must be 16-byte aligned"),
    (dict(cache_seqlens=A["cache_seqlens"] + 2), "cache_seqlens must be 4-byte aligned"),
    (dict(seqlens_out=A["seqlens_out"] + 1), "seqlens_out must be 4-byte aligned"),
    (dict(k_new=A["k_cache"] + 64), "k_cache overlaps k_new"),
    (dict(q=A["v_cache"]), "v_cache overlaps q"),
    (dict(q_out=A["k_new"] + 16), "q_out overlaps k_new"),
    (dict(q_out=A["q"] + 16), "q_out overlaps q"),
    (dict(seqlens_out=A["cache_seqlens"] + 4), "seqlens_out overlaps cache_seqlens"),
    (dict(v_cache=A["k_cache"] + 1024), "k_cache overlaps v_cache"),
]


@pytest.mark.parametrize("T", ["f16", "bf16"])
@pytest.mark.parametrize("paged", [False, True], ids=["dense", "paged"])
@pytest.mark.parametrize("kw,text", BAD)
def test_c_rejects(built_lib, T, paged, kw, text):
    kw = dict(kw)
    if "cache_dtype" in kw and T == "bf16" and kw["cache_dtype"] != 3:
        kw["cache_dtype"] = {2: 1, 0: 0}[kw["cache_dtype"]]
        text = text.replace("must be 1", "must be 2").replace("=2 ", "=1 ")
    if T == "bf16" and "cache_dtype" not in kw:
        kw["cache_dtype"] = 2
    assert _call(built_lib, T, paged, **kw) == -1
    err = _capi.last_error()
    assert err.startswith("kvcache_append: ") and text in err, err


PAGED_BAD = [
    (dict(block_table=None), "block_table is NULL"), (dict(num_pages=0), "num_pages=0 must be >= 1"),
    (dict(page_size=0), "page_size=0 must be >= 1"), (dict(max_pages_per_seq=0), "max_pages_per_seq=0 must be >= 1"),
    (dict(page_size=8), "page_size=8 must be a power of two >= 16"),
    (dict(page_size=48), "page_size=48 must be a power of two >= 16"),
    (dict(block_table=A["block_table"] + 2), "block_table must be 4-byte aligned"),
    (dict(seqlens_out=A["block_table"] + 4), "seqlens_out overlaps block_table"),
    (dict(rotary_len=67), "rotary_len=67 must be >= capacity + n_new = 68"),
    (dict(max_pages_per_seq=2 ** 27, rotary_len=2 ** 31 - 1), "capacity 2147483648 + n_new 4 positions exceed"),
]


@pytest.mark.parametrize("T", ["f16", "bf16"])
@pytest.mark.parametrize("kw,text", PAGED_BAD)
def test_c_rejects_paged(built_lib, T, kw, text):
    assert _call(built_lib, T, True, cache_dtype=1 if T == "f16" else 2, **kw) == -1
    err = _capi.last_error()
    assert text in err, err


@pytest.mark.parametrize("kw,text", [(dict(rotary_len=67), "rotary_len=67 must be >= capacity + n_new = 68"),
                                     (dict(Nk=0), "Nk=0 must be >= 1"),
                                     (dict(Nk=2 ** 31 - 3, rotary_len=2 ** 31 - 1), "positions exceed 2^31 - 1"),
                                     (dict(B=2 ** 20, n_new=2 ** 10, H=2 ** 4, Hkv=2), "rows, at most 2^31 - 1")])
def test_c_rejects_dense(built_lib, kw, text):
    assert _call(built_lib, "f16", False, **kw) == -1
    assert text in _capi.last_error(), _capi.last_error()


@pytest.mark.parametrize("which", ["k_scale", "v_scale"])
@pytest.mark.parametrize("value", [0.0, -0.0, -1.0, math.nan, math.inf, -math.inf])
def test_c_scales_finite_and_positive(built_lib, which, value):
    assert _call(built_lib, cache_dtype=3, **{which: value}) == -1
    err = _capi.last_error()
    assert err.startswith(f"kvcache_append: {which}=") and err.endswith("must be finite and > 0"), err


# ------------------------------------------------------------------ Python
def _t(*shape, dtype=torch.float16):
    return torch.zeros(*shape, dtype=dtype)


def _py(**kw):
    a = dict(k=_t(2, 2, 4, 64), v=_t(2, 2, 4, 64), k_cache=_t(2, 2, 64, 64), v_cache=_t(2, 2, 64, 64),
             cache_seqlens=torch.zeros(2, dtype=torch.int32))
    a.update(kw)
    n0 = _capi.launch_count()
    try:
        flash_attn.kvcache_append(a.pop("k"), a.pop("v"), a.pop("k_cache"), a.pop("v_cache"), a.pop("cache_seqlens"),
                                  **a)
    finally:
        assert _capi.launch_count() == n0


E4 = torch.float8_e4m3fn
PY_BAD = [
    (dict(k=None), "k must be a torch.Tensor"),
    (dict(v=_t(2, 2, 4, 64, dtype=torch.bfloat16)), "k and v must share one dtype"),
    (dict(k=_t(2, 2, 4, 64, dtype=torch.float32), v=_t(2, 2, 4, 64, dtype=torch.float32)), "fp16 or bf16"),
    (dict(k_cache=_t(2, 2, 64, 64, dtype=torch.bfloat16)), "k_cache and v_cache must both have k's dtype"),
    (dict(k_cache=_t(2, 2, 64, 64, dtype=E4)), "k_cache and v_cache must both have k's dtype"),
    (dict(v=_t(2, 2, 5, 64)), "k and v must be [B, Hkv, n_new, D] of one shape"),
    (dict(k_cache=_t(2, 2, 64, 32)), "k_cache and v_cache must be [B, Hkv, Nk, D]"),
    (dict(block_table=torch.zeros(2, 4, dtype=torch.int32), k_cache=_t(10, 24, 2, 64), v_cache=_t(10, 24, 2, 64)),
     "page_size (k_cache.shape[1]) must be a power of two >= 16"),
    (dict(block_table=torch.zeros(2, 4, dtype=torch.int32), k_cache=_t(10, 16, 3, 64), v_cache=_t(10, 16, 3, 64)),
     "must be pools [num_pages, page_size, Hkv, D]"),
    (dict(block_table=torch.zeros(3, 4, dtype=torch.int32), k_cache=_t(10, 16, 2, 64), v_cache=_t(10, 16, 2, 64)),
     "block_table must be an int32"),
    (dict(q=_t(2, 3, 4, 64)), "q must be [B, H, n_new, D]"),
    (dict(q=_t(2, 4, 4, 64), q_out=_t(2, 4, 4, 32)), "q_out must have q's shape and dtype"),
    (dict(q_out=_t(2, 4, 4, 64)), "q_out needs q"),
    (dict(rotary_cos=torch.zeros(68, 32)), "rotary_cos and rotary_sin must both be given"),
    (dict(rotary_cos=torch.zeros(68, 32, dtype=torch.float64), rotary_sin=torch.zeros(68, 32, dtype=torch.float64)),
     "must be fp32"),
    (dict(rotary_cos=torch.zeros(68, 12), rotary_sin=torch.zeros(68, 12)), "rotary_dim = 2 * rotary_cos.shape[1] = 24"),
    (dict(rotary_cos=torch.zeros(67, 32), rotary_sin=torch.zeros(67, 32)), "rotary_cos.shape[0] = 67 must be >= "
                                                                            "capacity + n_new = 68"),
    (dict(rotary_interleaved=True), "rotary_interleaved needs rotary_cos"),
    (dict(k_scale=2.0), "k_scale=2.0 must be 1 unless the cache is float8_e4m3fn"),
    (dict(k_cache=_t(2, 2, 64, 64, dtype=E4), v_cache=_t(2, 2, 64, 64, dtype=E4), v_scale=math.inf),
     "v_scale=inf must be finite and > 0"),
    (dict(cache_seqlens=torch.zeros(3, dtype=torch.int32)), "cache_seqlens must be an int32"),
    (dict(seqlens_out=torch.zeros(2, dtype=torch.int64)), "seqlens_out must be an int32"),
    (dict(), "k must be a CUDA tensor on k's device"),
]


@pytest.mark.parametrize("kw,text", PY_BAD)
def test_python_rejects(kw, text):
    with pytest.raises(RuntimeError, match=re.escape(text)):
        _py(**kw)


@pytest.mark.parametrize("kw,text", [
    (dict(k=None), "k must be a torch.Tensor"),
    (dict(o=_t(2, 4, 4, 32)), "o must have q's shape"),
    (dict(q=_t(2, 4, 4, 64, dtype=torch.bfloat16), o=_t(2, 4, 4, 64, dtype=torch.bfloat16)), "q must be"),
    (dict(q=_t(2, 3, 4, 64), o=_t(2, 3, 4, 64)), "Hkv dividing H"),
    (dict(num_splits=65), "num_splits must be an int"),
    (dict(lse=torch.zeros(2, 4, 5)), "lse must be"),
    (dict(), "must be a CUDA tensor"),
])
def test_python_fused_rejects(kw, text):
    a = dict(q=_t(2, 4, 4, 64), k_cache=_t(2, 2, 64, 64), v_cache=_t(2, 2, 64, 64), o=_t(2, 4, 4, 64),
             k=_t(2, 2, 4, 64), v=_t(2, 2, 4, 64), cache_seqlens=torch.zeros(2, dtype=torch.int32))
    a.update(kw)
    n0 = _capi.launch_count()
    with pytest.raises(RuntimeError, match=text):
        flash_attn.fmha_fwd_kvcache(a.pop("q"), a.pop("k_cache"), a.pop("v_cache"), a.pop("o"), a.pop("k"),
                                    a.pop("v"), a.pop("cache_seqlens"), **a)
    assert _capi.launch_count() == n0
