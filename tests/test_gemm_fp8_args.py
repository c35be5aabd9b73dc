"""Argument checks of the fp8 GEMM: the C entry b200_gemm_e4m3 and hgemm.scaled_mm reject every bad argument on the
host, with a message naming it, before any CUDA call and without a launch (_capi.launch_count() unchanged).  No GPU
needed: the C pointers are fake addresses that are never dereferenced, and the Python checks run on CPU tensors."""
import re

import pytest
import torch

from leetcuda_b200 import _capi, hgemm

A = {n: (i + 1) << 32 for i, n in enumerate(["a", "b", "c", "sa", "sb"])}
GOOD = dict(M=256, N=256, K=256, recipe=0, dtype=1)


def _call(lib, **kw):
    x = dict(A, **GOOD)
    x.update(kw)
    n0 = _capi.launch_count()
    rc = lib.b200_gemm_e4m3(x["a"], x["b"], x["c"], x["sa"], x["sb"], x["M"], x["N"], x["K"], x["recipe"], x["dtype"],
                            None)
    assert _capi.launch_count() == n0
    return rc


BAD = [
    (dict(a=None), "a is NULL"), (dict(b=None), "b_nk is NULL"), (dict(c=None), "c is NULL"),
    (dict(sa=None), "scale_a is NULL"), (dict(sb=None), "scale_b is NULL"),
    (dict(a=A["a"] + 8), "a must be 16-byte aligned"), (dict(b=A["b"] + 4), "b_nk must be 16-byte aligned"),
    (dict(c=A["c"] + 2), "c must be 16-byte aligned"), (dict(sa=A["sa"] + 2), "scale_a must be 4-byte aligned"),
    (dict(sb=A["sb"] + 1), "scale_b must be 4-byte aligned"),
    (dict(M=0), "M=0 must be >= 1"), (dict(N=-8), "N=-8 must be >= 1"), (dict(K=0), "K=0 must be >= 1"),
    (dict(K=136), "K=136 must be a multiple of 16"), (dict(N=260), "N=260 must be a multiple of 8"),
    (dict(recipe=3), "scale_recipe=3 must be"), (dict(recipe=-1), "scale_recipe=-1 must be"),
    (dict(dtype=0), "c_dtype=0 must be B200_DTYPE_F16"), (dict(dtype=3), "c_dtype=3 must be B200_DTYPE_F16"),
    (dict(c=A["a"] + 256 * 255), "c overlaps a"), (dict(c=A["b"] - 16), "c overlaps b_nk"),
    (dict(sa=A["c"] + 1024), "c overlaps scale_a"),
    (dict(recipe=2, sb=A["c"] + 256 * 256 * 2 - 4), "c overlaps scale_b"),
]


@pytest.mark.parametrize("kw,text", BAD)
def test_c_rejects(built_lib, kw, text):
    assert _call(built_lib, **kw) == -1
    err = _capi.last_error()
    assert err.startswith("gemm_e4m3: ") and text in err, err


def test_c_scale_extent_follows_the_recipe(built_lib):
    """scale_b 400 bytes before c: one value (tensor) ends before c, N values (row) reach into it."""
    assert _call(built_lib, sb=A["c"] - 400, recipe=1) == -1 and "c overlaps scale_b" in _capi.last_error()


# ------------------------------------------------------------------ Python
E4 = torch.float8_e4m3fn


def _args(M=64, N=136, K=256, recipe="tensor"):
    a = torch.zeros(M, K, dtype=E4)
    b = torch.zeros(N, K, dtype=E4).t()
    c = torch.zeros(M, N, dtype=torch.float16)
    kbs, nbs = -(-K // 128), -(-N // 128)
    sa = {"tensor": torch.ones(1), "row": torch.ones(M, 1), "block": torch.ones(kbs, M).t()}[recipe]
    sb = {"tensor": torch.ones(1), "row": torch.ones(1, N), "block": torch.ones(nbs, kbs)}[recipe]
    return dict(a=a, b=b, c=c, scale_a=sa, scale_b=sb, scale_recipe=recipe)


def _py(**kw):
    x = _args(recipe=kw.pop("recipe", "tensor"))
    x.update(kw)
    n0 = _capi.launch_count()
    try:
        hgemm.scaled_mm(x.pop("a"), x.pop("b"), x.pop("c"), x.pop("scale_a"), x.pop("scale_b"), **x)
    finally:
        assert _capi.launch_count() == n0


_buf = torch.zeros(64 * 136 * 2 + 64, dtype=torch.uint8)
PY_BAD = [
    (dict(a=None), "a must be a torch.Tensor"),
    (dict(scale_b=2.0), "scale_b must be a torch.Tensor"),
    (dict(bias=torch.zeros(136)), "bias is not supported"),
    (dict(scale_recipe="channel"), "scale_recipe must be 'tensor', 'row' or 'block'"),
    (dict(a=torch.zeros(64, 256, dtype=torch.float8_e5m2)), "a must be torch.float8_e4m3fn"),
    (dict(b=torch.zeros(136, 256, dtype=torch.float8_e5m2).t()), "e5m2 and other fp8 formats are not supported"),
    (dict(a=torch.zeros(64, 256, dtype=torch.float16)), "a must be torch.float8_e4m3fn (e4m3), got torch.float16"),
    (dict(c=torch.zeros(64, 136, dtype=torch.float32)), "c must be torch.float16 or torch.bfloat16, got torch.float32"),
    (dict(c=torch.zeros(64, 136, dtype=E4)), "c must be torch.float16 or torch.bfloat16"),
    (dict(b=torch.zeros(256, 136, dtype=E4)), "b must be column-major"),
    (dict(a=torch.zeros(256, 64, dtype=E4).t()), "a must be contiguous"),
    (dict(c=torch.zeros(136, 64, dtype=torch.float16).t()), "c must be contiguous"),
    (dict(c=torch.zeros(64, 128, dtype=torch.float16)), "do not form [M,K] x [K,N] -> [M,N]"),
    (dict(b=torch.zeros(136, 128, dtype=E4).t()), "do not form"),
    (dict(a=torch.zeros(2, 64, 256, dtype=E4)), "must be 2-D"),
    (dict(scale_a=torch.ones(1, dtype=torch.float64)), "scale_a must be torch.float32"),
    (dict(scale_a=torch.ones(2)), "tensor scaling takes one scale_a and one scale_b value"),
    (dict(recipe="row", scale_a=torch.ones(1, 64)), "row scaling takes a contiguous scale_a of shape [64]"),
    (dict(recipe="row", scale_b=torch.ones(136, 1)), "row scaling takes a contiguous scale_b of shape [136]"),
    (dict(recipe="block", scale_a=torch.ones(64, 2)), "block scaling takes scale_a [64, 2] with stride (1, 64)"),
    (dict(recipe="block", scale_a=torch.ones(64, 3)), "block scaling takes scale_a [64, 2]"),
    (dict(recipe="block", scale_b=torch.ones(2, 3)), "block scaling takes scale_b [2, 2] row-major"),
    (dict(recipe="block", scale_b=torch.ones(2, 2).t()[:, :1].expand(2, 2)), "block scaling takes scale_b"),
    (dict(c=_buf[:64 * 136 * 2].view(torch.float16).view(64, 136),
          scale_a=_buf[64 * 136 * 2 - 4:64 * 136 * 2].view(torch.float32)), "c overlaps scale_a"),
    (dict(), "a must be a CUDA tensor"),
]


@pytest.mark.parametrize("kw,text", PY_BAD)
def test_python_rejects(kw, text):
    with pytest.raises(RuntimeError, match=re.escape(text)):
        _py(**kw)


def test_python_overlap_with_operands():
    x = _args()
    buf = torch.zeros(64 * 136 * 2, dtype=torch.uint8)
    n0 = _capi.launch_count()
    with pytest.raises(RuntimeError, match="c overlaps a"):
        hgemm.scaled_mm(buf[:64 * 256].view(E4).view(64, 256), x["b"], buf.view(torch.float16).view(64, 136),
                        x["scale_a"], x["scale_b"], scale_recipe="tensor")
    assert _capi.launch_count() == n0


def test_exported():
    assert "scaled_mm" in hgemm.__all__
    assert _capi.SCALE_TENSOR == 0 and _capi.SCALE_ROW == 1 and _capi.SCALE_BLOCK == 2
