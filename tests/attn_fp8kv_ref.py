"""fp8 (e4m3) K/V attention (b200_fmha_fwd_{f16,bf16}_fp8kv_{seqlens,paged}, flash_attn.fmha_fwd with float8_e4m3fn K
and V): the dispatch restated on the CPU, the quantisation and the exact e4m3 -> T conversion, the per-element bound,
and the GPU case table.  Used by test_attn_fp8kv_coverage.py, test_attn_fp8kv_sharpness.py and test_attn_fp8kv_gpu.py.

Dispatch.  An fp8 call runs attn_fwd_fp8kv_seqlens_kernel (a dense call: null length arrays) or, with a block table,
attn_fwd_fp8kv_paged_kernel, each with the template arguments and tiling of the fp16 / bf16 seqlens and paged kernels
and the element type T of Q and O as its last argument.  So a path key is (T,) + attn_bf16_ref's key, and num_splits = 0
resolves from the padded shape, b200_fmha_fwd_f16_gqa_splits, as for the T calls.

Arithmetic.  K and V codes are widened exactly to T (every finite e4m3 value is an fp16 and a bf16 value); the softmax
scale is c = fp32(scale * k_scale); the kernel is then the T kernel on those K and V, up to its fp32 O, which is
multiplied by v_scale in fp32 and rounded once to T (split: each part's fp32 O is multiplied before the combine).

Bound.  The truth is fp64 attention on the dequantised K and V: O* = v_scale * softmax(scale * k_scale * Q K^T) V with K,
V the code values.  Against it, per element:
  * the T kernel's bound on the code values with the kernel's scale c (attn_ref.o_bound for fp16, attn_bf16_ref.o_bound
    for bf16, without the final rounding; split: the combine bounds), times v_scale;
  * the scale fold: c = scale * k_scale * (1 + d), |d| <= 2^-24, moves every score x_j = c s_j by |d x_j| and a weight by
    at most e^(2 |d| max_j |x_j|) - 1 <= 4 |d| max_j |x_j| relative, so O by that times (sigma + |O|) (attn_ref's weight
    term) and lse by |d| max_j |x_j|;
  * the v_scale multiply: one fp32 rounding, 2^-24 of v_scale (|O| + pre) (split: of every part, at most the column's
    largest |V| of the code values, 2^-23 v_scale max|V| covers it);
  * O's rounding to T: u_T (v_scale |O| + the terms above) plus T's smallest-spacing floor (taken unscaled);
  * masked keys: a key whose exponential runs on the FMA pipe gets P = 2^-126 instead of 0 when it is masked
    (exp2_fma_pipe(-inf), attn_sm90.cuh).  fp16's rounding of P flushes it; bf16 keeps it, so O moves by at most
    2^-126 sum_j |v_j| over the keys of the visited blocks (l >= 1), which 2^-126 N 448 v_scale covers (N the padded
    keys, 448 the largest code).  Only rows whose visible V is ~0 can tell.
lse does not see v_scale.  Nothing is fitted.
"""
from __future__ import annotations

import math
import re
from collections import namedtuple

import numpy as np
import torch

import attn_bf16_ref as BF
import attn_paged_ref as P
import attn_ref as R
import attn_seqlens_ref as S
import attn_split_ref as SR

TYPES = ("half", "bf16")
TORCH = {"half": torch.float16, "bf16": torch.bfloat16}
MANGLED_T = {"6__half": "half", "13__nv_bfloat16": "bf16", "__half": "half", "__nv_bfloat16": "bf16"}
U = {"half": R.U16, "bf16": BF.U8}
FLOOR = {"half": 2.0 ** -24, "bf16": BF.O_FLOOR}
E4M3_MAX = 448.0
DELTA = 2.0 ** -24   # the fp32 roundings of scale * k_scale and of O * v_scale
LEAK = 2.0 ** -126 * E4M3_MAX   # per key: a masked key's P = 2^-126 times the largest |V|


# ------------------------------------------------------------------ the dispatch
def path(kind, T, B, H, Hkv, Nq, Nk, D, causal, splits, page_size=None):
    """(path key, launches) of an fp8 call with Q/O type T ("half" or "bf16"): kind "dense", "seqlens" or "paged"."""
    if D % 16:
        raise ValueError(f"fp8 K/V need D % 16 == 0, got D{D}")
    key, n = BF.path(kind, B, H, Hkv, Nq, Nk, D, causal, splits, page_size)
    return (T,) + key, n


def instantiation(key):
    """(kernel, kDS, kBN, kWG, kCausal, kSplit, T) of a path key."""
    return key[1:7] + (key[0],)


def reachable():
    """Every path key: the bf16 paths (the fp16 seqlens and paged paths) for either Q/O type."""
    return {(T,) + k for T in TYPES for k in BF.reachable()}


_MANGLED = re.compile(r"attn_fwd_fp8kv_(seqlens|paged)_kernelILi(\d+)ELi(\d+)ELi(\d+)ELb([01])ELb([01])E"
                      r"(6__half|13__nv_bfloat16)E")
_DEMANGLED = re.compile(r"attn_fwd_fp8kv_(seqlens|paged)_kernel<(\d+), (\d+), (\d+), (true|false), (true|false), "
                        r"(__half|__nv_bfloat16)>")


def parse_instantiations(names):
    out = []
    for name in names:
        for m in list(_MANGLED.finditer(name)) + list(_DEMANGLED.finditer(name)):
            a = m.groups()
            out.append((a[0], int(a[1]), int(a[2]), int(a[3]), *(x in ("1", "true") for x in a[4:6]),
                        MANGLED_T[a[6]]))
    return out


# ------------------------------------------------------------------ e4m3
def finite_codes():
    """The 254 finite e4m3 codes (every byte but 0x7F and 0xFF, the NaNs) as uint8."""
    return torch.tensor([c for c in range(256) if c & 0x7F != 0x7F], dtype=torch.uint8)


def decode(codes):
    """Exact values of e4m3 codes (uint8 tensor, any device) as fp64, from the format's definition."""
    c = codes.to(torch.int64)
    sign = torch.where(c >= 128, -1.0, 1.0).double()
    e, m = (c >> 3) & 15, (c & 7).double()
    val = torch.where(e == 0, m * 2.0 ** -9, (8 + m) * torch.pow(2.0, (e - 10).double()))
    val = torch.where((c & 0x7F) == 0x7F, torch.full_like(val, float("nan")), val)
    return (sign * val).to(codes.device)


def quantise(x, scale):
    """e4m3 codes (float8_e4m3fn) of x / scale, clamped to +-448 (what a cache writer stores)."""
    return (x.float() / scale).clamp(-E4M3_MAX, E4M3_MAX).to(torch.float8_e4m3fn)


def widen(x8, T):
    """The kernel's conversion of e4m3 codes to T: exact, so torch's conversion is it."""
    return x8.to(TORCH[T])


# ------------------------------------------------------------------ the bound
def score_max(q, k, scale):
    """max_j |scale q_i . k_j| per row (fp64; q [..., Nq, D], k [..., Nk, D] with matching leading dims)."""
    if isinstance(q, torch.Tensor):
        return (q.double().abs() @ k.double().abs().transpose(-1, -2)).amax(-1) * scale
    return (np.abs(np.asarray(q, np.float64)) @ np.abs(np.asarray(k, np.float64)).T).max(-1) * scale


def o_bound(ref, poly, T, v_scale, xmax):
    """Bound of the kernel's O against v_scale * O(exact scale) per element; ref: the reference at the kernel's scale
    on the code values; xmax: score_max at the kernel's scale."""
    pre = (BF.o_bound(ref, poly) if T == "bf16" else R.o_bound(ref, poly))[0]
    ao = abs(ref["o"])
    fold = 4 * DELTA * xmax[..., None] * (ref["sigma"] + ao)
    b = v_scale * (pre + fold + LEAK * ref["N"]) + DELTA * v_scale * (ao + pre + fold)
    return b + U[T] * (v_scale * ao + b) + FLOOR[T]


def lse_bound(ref, poly, xmax):
    return R.lse_bound(ref, poly) + DELTA * xmax


def combine_bound(parts, poly, T, v_scale, xmax, vmax):
    """(O at the kernel's scale, L, empty, O bound, lse bound) of a split row against v_scale * O(exact scale); vmax:
    the largest |V| code value per column, broadcastable to O."""
    o, L, empty, ob, lb = (BF.combine_bound if T == "bf16" else SR.combine_bound)(parts, poly)
    sigma = sum(p["sigma"] for p in parts)   # >= the combined row's sigma
    fold = 4 * DELTA * xmax[..., None] * (sigma + abs(o))
    leak = LEAK * parts[0]["N"]
    return (o, L, empty, v_scale * (ob + fold + leak) + FLOOR[T] + 2 * DELTA * v_scale * (vmax + fold),
            lb + DELTA * xmax)


# ------------------------------------------------------------------ CPU restatement
def kernel_o(q, k8, v8, scale, k_scale, v_scale, kbn, T, poly_mask=0, k_first=False, v_after=False):
    """The fp8 kernel's arithmetic on one head (q [N, D] numpy of T values, k8 / v8 float8_e4m3fn CPU tensors): O as
    fp32 holding T values.  The wrong designs: k_first multiplies K by k_scale and rounds it to T (the scale unfolded),
    v_after multiplies the rounded O by v_scale and rounds again."""
    if k_first:
        k = (k8.to(torch.float32) * k_scale).to(TORCH[T]).float().numpy()
        c = float(np.float32(scale))
    else:
        k = k8.to(TORCH[T]).float().numpy()
        c = float(np.float32(np.float32(scale) * np.float32(k_scale)))
    v = v8.to(TORCH[T]).float().numpy()
    o, lse = BF.online(q, k, v, c, kbn, poly_mask, p_round="f16" if T == "half" else "rn", o_round=None)
    rnd = (lambda x: x.astype(np.float16).astype(np.float32)) if T == "half" else BF.round_bf16
    if v_after:
        return rnd((rnd(o) * np.float32(v_scale)).astype(np.float32)), lse
    return rnd((o * np.float32(v_scale)).astype(np.float32)), lse


# ------------------------------------------------------------------ the GPU case table
def fp8_dim(D):
    """The case tables' head dim rounded up to a multiple of 16 inside its kernel family (and slab count): 520, 776
    and 1000 become 528 (a last slab of one 16-column chunk), 784 and 1008 (a last K chunk of 48 columns), where the
    fp8 ring of 12, 10 and 8 slots holds less than one key block (attn_ring_ref)."""
    return -(-D // 16) * 16


def _cases():
    out = []
    for kind, c in BF.CASES:
        if kind == "dense" and c.D == 264:
            continue   # fp8_dim would make it D 272, already covered by the seqlens / paged rows
        out.append((kind, c._replace(D=fp8_dim(c.D))))
    return out


Scales = namedtuple("Scales", "k v")
# a large v_scale keeps 448 v_scale inside fp16's range (65504)
SCALES = [Scales(1.0, 1.0), Scales(0.25, 4.0), Scales(0.37, 0.37), Scales(300.0, 100.0)]
_ROWS = [(T, kind, c) for T in TYPES for kind, c in _cases()]
# the rows of head dims > 512 (attn_ring_ref's regimes) last, so that the others keep their places
CASES = [x for x in _ROWS if x[2].D <= 512] + [x for x in _ROWS if x[2].D > 512]


def case_key(T, kind, c):
    if kind == "paged":
        return path("paged", T, len(c.lq), c.H, c.Hkv, c.Nq, c.page_size * c.max_pages, c.D, c.causal, c.splits,
                    c.page_size)[0]
    if kind == "seqlens":
        return path("seqlens", T, len(c.lq), c.H, c.Hkv, c.Nq, c.Nk, c.D, c.causal, c.splits)[0]
    return path("dense", T, 2, c.H, c.Hkv, c.Nq, c.Nk, c.D, c.causal, c.splits)[0]
