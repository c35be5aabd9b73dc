"""bf16 attention (b200_fmha_fwd_bf16_seqlens / _paged, flash_attn.fmha_fwd on bf16 tensors): the dispatch restated on the
CPU, the per-element bound with bf16 roundings, and the GPU case table.  Used by test_attn_bf16_coverage.py,
test_attn_bf16_sharpness.py and test_attn_bf16_gpu.py.

Dispatch.  Every bf16 call runs attn_fwd_seqlens_bf16_kernel (a dense call: null length arrays, so every sequence has
Nq queries and Nk keys) or, with a block table, attn_fwd_paged_bf16_kernel.  Their template arguments and tilings are
those of the fp16 seqlens and paged kernels, so a path key is ("seqlens",) + attn_seqlens_ref's key or ("paged",) +
attn_paged_ref's key, and the split count of num_splits = 0 is b200_fmha_fwd_f16_gqa_splits's, whatever the dtype.

Bound.  The kernel does what the fp16 kernel does (attn_ref.py) with two roundings changed: P is rounded to bf16
(cvt.rn.bf16x2.f32, nearest even) before P V and O is rounded once to bf16.  So attn_ref.o_bound holds with bf16's unit
roundoff u = 2^-8 in the places of U16:
  * P: u sigma (c = 1).  fp16's subnormal term 2^-25 tau (a P below 2^-14) has no bf16 counterpart of that size: bf16
    has fp32's exponent range, a P below 2^-126 is already flushed by ex2.approx.ftz in fp32 (absolute error < 2^-126
    per key), and bf16's subnormal grid is finer still.  2^-126 tau covers both and is negligible next to u sigma.
  * O: u |O64| plus half of bf16's smallest subnormal spacing, 2^-134 (for fp16 2^-24 covered its subnormals).
  * the weight errors, the fp32 sums and the accumulation are unchanged.  The score model rho carries over: a bf16 x bf16
    product, like an fp16 one, has at most 16 significant bits and is exact in fp32, and wgmma adds the products of a
    k16 step in fp32 the same way for both types.
lse does not see the roundings (m and l are fp32), so attn_ref.lse_bound holds unchanged.  A split row: attn_split_ref's
combine_bound with these part bounds and the final rounding to bf16.  The fp64 reference is computed from the bf16
inputs themselves (attn_ref.reference / attn_split_ref.masked_reference on the bf16 tensors).  Nothing is fitted.
"""
from __future__ import annotations

import math
import re
from collections import namedtuple

import numpy as np
import torch

import attn_mask_ref as M
import attn_paged_ref as P
import attn_ref as R
import attn_seqlens_ref as S

U8 = 2.0 ** -8                    # unit roundoff of bf16
FTZ = 2.0 ** -126                 # a P below fp32's normal range (ex2.approx.ftz) or on bf16's subnormal grid
O_FLOOR = 2.0 ** -134             # half of bf16's subnormal spacing


# ------------------------------------------------------------------ the dispatch
def path(kind, B, H, Hkv, Nq, Nk, D, causal, splits, page_size=None):
    """(path key, launches) of a bf16 call: kind "dense" (no lengths), "seqlens" or "paged" (Nk = max_pages *
    page_size)."""
    if kind == "paged":
        key, n = P.path(B, H, Hkv, Nq, page_size, Nk // page_size, D, causal, splits)
        return ("paged",) + key, n
    key, n = S.path(B, H, Hkv, Nq, Nk, D, causal, splits)
    return ("seqlens",) + key, n


def instantiation(key):
    """(kernel, kDS, kBN, kWG, kCausal, kSplit) of a path key."""
    return key[:6]


def reachable():
    """Every path key: the fp16 seqlens paths on the seqlens kernel, the fp16 paged paths on the paged kernel."""
    return {("seqlens",) + k for k in S.reachable()} | {("paged",) + k for k in P.reachable()}


_MANGLED = re.compile(r"attn_fwd_(seqlens|paged)_bf16_kernelILi(\d+)ELi(\d+)ELi(\d+)ELb([01])ELb([01])E")
_DEMANGLED = re.compile(r"attn_fwd_(seqlens|paged)_bf16_kernel<(\d+), (\d+), (\d+), (true|false), (true|false)>")


def parse_instantiations(names):
    out = []
    for name in names:
        for m in list(_MANGLED.finditer(name)) + list(_DEMANGLED.finditer(name)):
            a = m.groups()
            out.append((a[0], int(a[1]), int(a[2]), int(a[3]), *(x in ("1", "true") for x in a[4:])))
    return out


# ------------------------------------------------------------------ the bound
def o_bound(ref, poly):
    """attn_ref.o_bound with bf16 roundings: (bound before O's rounding, bound of the bf16 O) per element."""
    N = ref["N"]
    acc = (math.ceil(N / 16) + 16 + math.ceil(N / 64)) * 2.0 ** -23
    ao = abs(ref["o"])
    pre = ((U8 + acc) * ref["sigma"] + R._weight_err(ref, poly) * (ref["sigma"] + ao) + R._lsum_err(N) * ao
           + FTZ * ref["tau"])
    return pre, pre + U8 * ao + O_FLOOR


lse_bound = R.lse_bound


def combine_bound(parts, poly):
    """attn_split_ref.combine_bound with the parts' bf16 pre-rounding bounds and the final rounding to bf16: (O*, L*,
    empty, O bound, lse bound)."""
    is_t = isinstance(parts[0]["o"], torch.Tensor)
    xp = torch if is_t else np
    S_ = len(parts)
    lse = xp.stack([p["lse"] for p in parts])
    top = lse.amax(0) if is_t else lse.max(axis=0)
    empty = xp.isinf(top)
    topf = xp.where(empty, 0.0, top)
    W = xp.exp(lse - topf)
    W = W / xp.where(empty, 1.0, W.sum(0))
    L = xp.where(empty, -math.inf, topf + xp.log(xp.where(empty, 1.0, xp.exp(lse - topf).sum(0))))
    pe = [p["empty"] for p in parts]
    e = xp.stack([xp.where(pe[z], 0.0, lse_bound(parts[z], poly)) for z in range(S_)])
    delta = xp.where(xp.stack(pe), 0.0, topf - lse)
    a0 = e + 2.0 ** -22 + 2.0 ** -24
    A0 = a0.amax(0) if is_t else a0.max(axis=0)
    a = a0 + 2.0 ** -24 * (delta + 2 * A0)
    A = a.amax(0) if is_t else a.max(axis=0)
    o = sum(W[z][..., None] * parts[z]["o"] for z in range(S_))
    term1 = term2 = term3 = 0.0
    for z in range(S_):
        pre = xp.where(pe[z][..., None], 0.0, o_bound(parts[z], poly)[0])
        g = (W[z] * xp.exp(a[z] + A))[..., None]
        term1 = term1 + g * pre
        term2 = term2 + g * (a[z] + A)[..., None] * abs(parts[z]["o"] - o)
        term3 = term3 + g * (abs(parts[z]["o"]) + pre)
    pre_all = term1 + term2 + (3 * S_ + 2) * 2.0 ** -24 * term3
    ob = pre_all + U8 * (abs(o) + pre_all) + O_FLOOR
    lb = A + (S_ + 1) * 2.0 ** -24 + 2.0 ** -22 * (math.log(S_) + 1) + 2.0 ** -24 * abs(xp.where(empty, 0.0, L))
    return o, L, empty, ob, lb


# ------------------------------------------------------------------ CPU restatement of the bf16 roundings
def round_bf16(x, mode="rn"):
    """fp32 values rounded to bf16 (returned as fp32): "rn" nearest even (cvt.rn.bf16x2.f32), "rz" truncation."""
    u = np.ascontiguousarray(x, np.float32).view(np.uint32).astype(np.uint64)
    if mode == "rn":
        u = u + 0x7FFF + ((u >> 16) & 1)
    return (u & 0xFFFF0000).astype(np.uint32).view(np.float32)


def online(q, k, v, scale, kbn, poly_mask=0, p_round="rn", o_round="rn"):
    """The kernel's bf16 arithmetic on one head ([N, D] numpy holding bf16 values): attn_ref.online(kernel=True) with P
    and O rounded to bf16 (`p_round` / `o_round`: "rn", "rz", or "f16" for an fp16 rounding).  Returns (O fp32, lse)."""
    ft = np.float32
    c = ft(ft(scale) * ft(R.LOG2E))
    s_all = q.astype(ft) @ k.astype(ft).T
    n, nk = q.shape[0], k.shape[0]
    m = np.full((n, 1), -np.inf, ft)
    l = np.zeros((n, 1), ft)
    o = np.zeros((n, v.shape[1]), ft)
    rnd = {"f16": lambda x: x.astype(np.float16).astype(ft), "rn": round_bf16,
           "rz": lambda x: round_bf16(x, "rz"), None: lambda x: x}
    with np.errstate(invalid="ignore", over="ignore"):
        for b0 in range(0, nk, kbn):
            s = s_all[:, b0:b0 + kbn]
            mn = np.maximum(m, (s.max(axis=1, keepdims=True) * c).astype(ft))
            alpha = np.exp2(m - mn).astype(ft)
            x = (s.astype(np.float64) * np.float64(c) - mn).astype(ft)
            p = np.exp2(x).astype(ft)
            if poly_mask:
                pair = (np.arange(b0, b0 + s.shape[1]) % 32) // 2
                sel = ((poly_mask >> pair) & 1).astype(bool)
                p[:, sel] = R.exp2_fma_pipe(x[:, sel])
            m = mn
            l = (l * alpha + p.sum(axis=1, keepdims=True)).astype(ft)
            o = (o * alpha + rnd[p_round](p) @ v[b0:b0 + kbn].astype(ft)).astype(ft)
    o = (o * (ft(1) / l)).astype(ft)
    lse = ((m + np.log2(l)) * ft(math.log(2.0)))[:, 0]
    return rnd[o_round](o), lse


def online_split(q, k, v, scale, kbn, splits, poly_mask=0, part_round=None):
    """Split-KV of one head: the key blocks cut into `splits` contiguous ranges (attn_split_ref.split_ranges), fp32
    parts, the combine's expf / fmaf / reciprocal and one rounding to bf16.  part_round="rn" restates the mistake of
    rounding every part to bf16 before the combine (O rounded twice)."""
    ft = np.float32
    nkv = -(-k.shape[0] // kbn)
    po, pl = [], []
    for b, e in [(nkv * z // splits, nkv * (z + 1) // splits) for z in range(splits)]:
        o, lse = online(q, k[b * kbn:e * kbn], v[b * kbn:e * kbn], scale, kbn, poly_mask, o_round=part_round)
        po.append(o.astype(ft))
        pl.append(lse.astype(ft))
    pl = np.stack(pl)
    top = pl.max(axis=0)
    acc = np.zeros_like(po[0])
    den = np.zeros(top.shape, ft)
    for z in range(splits):
        w = np.exp((pl[z] - top).astype(ft)).astype(ft)
        den = (den + w).astype(ft)
        acc = (w[:, None].astype(np.float64) * po[z] + acc).astype(ft)
    res = (acc * (ft(1) / den)[:, None]).astype(ft)
    return round_bf16(res), (np.log(den).astype(ft) + top).astype(ft)


# ------------------------------------------------------------------ the GPU case table
# ("seqlens", attn_seqlens_ref's rows) and ("paged", attn_paged_ref's rows) reach every path key; the dense rows run the
# seqlens kernel without lengths: MHA and GQA, causal or not, one split, several, or the library's choice (0), at
# D = 40 .. 264 and at 1000 (four slabs, the smallest K/V ring: attn_ring_ref).
Dense = namedtuple("Dense", "H Hkv Nq Nk D causal splits gens")
DENSE = [
    Dense(4, 4, 257, 257, 64, False, 1, ("randn", "tail_max")),
    Dense(8, 2, 200, 330, 128, True, 1, ("randn", "diag_gather")),
    Dense(8, 8, 130, 130, 264, True, 1, ("randn", "future_max")),
    Dense(8, 1, 1, 4100, 128, False, 0, ("randn", "front_max")),
    Dense(8, 2, 5, 777, 40, True, 3, ("randn", "diag_gather")),
    Dense(4, 2, 130, 300, 136, False, 2, ("randn", "one_hot")),
    Dense(8, 2, 130, 330, 1000, True, 1, ("randn", "future_max")),
    Dense(4, 1, 1, 1000, 1000, False, 4, ("randn", "tail_max")),
]
_ROWS = ([("seqlens", c) for c in S.CASES_BY_SHAPE] + [("paged", c) for c in P.CASES_BY_SHAPE]
         + [("dense", c) for c in DENSE])
# the rows of head dims > 512 (attn_ring_ref's regimes) last, so that the others keep their places
CASES = [x for x in _ROWS if x[1].D <= 512] + [x for x in _ROWS if x[1].D > 512]


def case_key(kind, c, splits=None):
    if kind == "paged":
        return path("paged", len(c.lq), c.H, c.Hkv, c.Nq, c.page_size * c.max_pages, c.D, c.causal, c.splits,
                    c.page_size)[0]
    if kind == "seqlens":
        return path("seqlens", len(c.lq), c.H, c.Hkv, c.Nq, c.Nk, c.D, c.causal, c.splits)[0]
    return path("dense", 2, c.H, c.Hkv, c.Nq, c.Nk, c.D, c.causal, c.splits if splits is None else splits)[0]


def exact_scores(gen):
    return M.exact_scores(gen)
