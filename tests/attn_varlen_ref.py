"""Packed variable-length attention (b200_fmha_fwd_{f16,bf16}_varlen and _varlen_paged, flash_attn.fmha_varlen_fwd):
the dispatch restated on the CPU, the packing of padded tensors into token-major ones and back, and the GPU case table.
Used by test_attn_varlen_coverage.py and test_attn_varlen_gpu.py.

Semantics.  q, o [total_q, H, D], k, v [total_k, Hkv, D]; sequence b has Lq_b = clamp(cu_q[b+1] - cu_q[b], 0, max_q)
queries at rows cu_q[b] + t and Lk_b = clamp(cu_k[b+1] - cu_k[b], 0, max_k) keys at rows cu_k[b] + t (paged K/V:
Lk_b = clamp(seqused_k[b], 0, max_pages * page_size), keys through the block table as in attn_paged_ref).  Everything
else is the seqlens call (attn_seqlens_ref) on padded [B, H, max_q, D] / [B, Hkv, max_k, D] copies, so pad() of the
packed tensors turns a varlen call into a seqlens (or paged) call with the same results, bit for bit.  Only the rows
cu_q[b] + t, t < Lq_b, inside [0, total_q) are written.

A path key is (kDS, kBN, kWG, kCausal, kPagedKV, T): the template arguments of attn_varlen_kernel.  Every query head
has tiles of its own (tph = ceil(max_q / (64 kWG)) of them), with or without the mask, so there is no tiling regime.
"""
from __future__ import annotations

import re
from collections import namedtuple

import attn_mask_ref as M
import attn_paths as P
import attn_ref as R

TYPES = {"fp16": "__half", "bf16": "__nv_bfloat16"}
_MANGLED_T = {"6__half": "__half", "13__nv_bfloat16": "__nv_bfloat16"}


# ------------------------------------------------------------------ the dispatch
def family(D):
    """(kDS, kBN, kWG) of attn_capi.cu's family(D)."""
    kbn, rows = M.kernel_shape(D)
    return P._SLAB[R.family(D)[0]], kbn, rows // 64


def path(H, Hkv, max_q, D, causal, paged, dtype):
    """The path key of one call (one launch, never split); dtype "fp16" or "bf16"."""
    if D % 8 or D > 1024 or H % Hkv or max_q < 1:
        raise ValueError(f"not a supported call: H{H} Hkv{Hkv} max_q{max_q} D{D}")
    return family(D) + (bool(causal), bool(paged), TYPES[dtype])


def tph(max_q, D):
    """Query tiles per query head."""
    _, _, wg = family(D)
    return -(-max_q // (64 * wg))


def grid(B, H, Hkv, max_q, D):
    """(grid.x, grid.y): G * tph * slabs CTAs per K/V head, B * Hkv K/V heads."""
    ds, _, _ = family(D)
    return (H // Hkv) * tph(max_q, D) * -(-D // ds), B * Hkv


def instantiation(key):
    return key


def name(inst):
    ds, bn, wg, causal, paged, t = inst
    return f"attn_varlen_kernel<{ds}, {bn}, {wg}, {str(causal).lower()}, {str(paged).lower()}, {t}>"


def reachable():
    """Every path key: the three kernel families, causal or not, packed or paged K/V, fp16 or bf16."""
    return {path(4, 2, 130, D, causal, paged, dt) for D in (40, 128, 264) for causal in (False, True)
            for paged in (False, True) for dt in TYPES}


INSTANTIATIONS = sorted(name(k) for k in reachable())

_MANGLED = re.compile(r"attn_varlen_kernelILi(\d+)ELi(\d+)ELi(\d+)ELb([01])ELb([01])E(6__half|13__nv_bfloat16)E")
_DEMANGLED = re.compile(r"attn_varlen_kernel<(\d+), (\d+), (\d+), (true|false), (true|false), (__half|__nv_bfloat16)>")


def parse_instantiations(names):
    out = []
    for n in names:
        for m in _MANGLED.finditer(n):
            a = m.groups()
            out.append((int(a[0]), int(a[1]), int(a[2]), a[3] == "1", a[4] == "1", _MANGLED_T[a[5]]))
        for m in _DEMANGLED.finditer(n):
            a = m.groups()
            out.append((int(a[0]), int(a[1]), int(a[2]), a[3] == "true", a[4] == "true", a[5]))
    return out


# ------------------------------------------------------------------ packing
def offsets(lens, first=0):
    """cu [B + 1] of raw lengths (the lengths a caller packs, which may exceed max_seqlen)."""
    cu = [first]
    for x in lens:
        cu.append(cu[-1] + int(x))
    return cu


def clamp(lens, n):
    return [min(max(int(x), 0), n) for x in lens]


def pack(x, cu, lens, total, fill):
    """Token-major [total, heads, D] of padded x [B, heads, N, D] (torch): rows cu[b] + t, t < lens[b] (clamped lengths)
    from x[b, :, t]; every other row `fill`."""
    import torch
    B, heads, _, D = x.shape
    out = torch.full((total, heads, D), fill, dtype=x.dtype, device=x.device)
    for b in range(B):
        n = lens[b]
        if n:
            out[cu[b]:cu[b] + n] = x[b, :, :n].transpose(0, 1)
    return out


def unpad_rows(o_pad, lse_pad, cu, lens):
    """[(row index of the packed output, o_pad[b, :, t] [H, D], lse_pad[b, :, t] [H])] of every owned row, stacked:
    (rows [n], o [n, H, D], lse [H, n])."""
    import torch
    rows, os_, ls = [], [], []
    for b, n in enumerate(lens):
        if n:
            rows.append(torch.arange(cu[b], cu[b] + n))
            os_.append(o_pad[b, :, :n].transpose(0, 1))
            ls.append(lse_pad[b, :, :n])
    return torch.cat(rows), torch.cat(os_), torch.cat(ls, dim=1)


# ------------------------------------------------------------------ the GPU case table
# One row per instantiation.  Every row's sequences (raw lengths, before the clamps) mix Lq 0, 1, short, long and one
# past max_q (its rows past max_q stay untouched); Lk 0, 1, kBN - 1, kBN + 1, one past max_k (paged: past the table's
# keys) and lengths that are not multiples of kBN; causal rows have Lq > Lk.  Head dims 8, 40, 64, 72, 128, 136, 256,
# 520 and 1024 (three and four slabs, a K/V ring shorter than one key block from 776 on); G in {1, 4, 8}.
Case = namedtuple("Case", "H Hkv D causal paged dtype lq lk max_q max_k page_size gens")

_DIMS = {64: (8, 64, 40), 128: (72, 128), 256: (136, 256, 520, 1024)}
_HEADS = [(4, 4), (8, 2), (8, 1)]
_ADVERSARIAL = [g for g in R.GENERATORS if g != "randn"]


def _rows():
    rows, n = [], 0
    for ds in (64, 128, 256):
        kbn = 128 if ds == 64 else 64
        for causal in (False, True):
            for paged in (False, True):
                for dt in TYPES:
                    dims = _DIMS[ds]
                    D = dims[n % len(dims)]
                    D = 40 if causal and D < 32 else D   # the diagonal probes need D >= 32 (attn_mask_ref)
                    H, Hkv = _HEADS[n % 3]
                    max_q, max_k = 130, 3 * kbn + 44
                    lq = (130, 0, 1, 77, 150, 5, 64)
                    lk = (kbn + 1, 5, 0, kbn - 1, max_k + 20, 3, 1)
                    ps = (16, kbn, 2 * kbn)[n % 3] if paged else None
                    gens = ("randn", _ADVERSARIAL[n % 5]) + ((M.PROBES[n % 2],) if causal else ())
                    rows.append(Case(H, Hkv, D, causal, paged, dt, lq, lk, max_q, max_k, ps, gens))
                    n += 1
    return rows


CASES_BY_SHAPE = _rows()
CASES = [(c, gen) for c in CASES_BY_SHAPE for gen in c.gens]


def case_key(c):
    return path(c.H, c.Hkv, c.max_q, c.D, c.causal, c.paged, c.dtype)


def cases_by_key(cases=None):
    out = {}
    for c, gen in (CASES if cases is None else cases):
        out.setdefault(case_key(c), []).append((c, gen))
    return out
