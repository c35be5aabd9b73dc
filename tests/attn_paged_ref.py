"""Paged K/V (b200_fmha_fwd_f16_paged): the dispatch, the kernel's sub-load addresses and the page gather restated on the
CPU, and the GPU case table.  Used by test_attn_paged_coverage.py and test_attn_paged_gpu.py.

Semantics.  k, v are pools [num_pages, page_size, Hkv, D]; key t of sequence b is row t % page_size of page
table[b][t // page_size].  Everything else is b200_fmha_fwd_f16_seqlens (attn_seqlens_ref) on the padded
Nk = max_pages * page_size, so gather() of the pools into a contiguous [B,Hkv,Nk,D] cache turns a paged call into a
seqlens call with the same results, bit for bit.

A path key is attn_seqlens_ref's key (kDS, kBN, kWG, kCausal, kSplit, tiling) followed by the page-size regime
"<", "=" or ">": page_size against kBN.  Below kBN a key block is kBN / page_size sub-loads from as many pages; at or
above it one sub-load, from inside a page ("=": the block is the page, ">": a block at an offset in it).
"""
from __future__ import annotations

import re
from collections import namedtuple

import attn_mask_ref as M
import attn_ref as R
import attn_seqlens_ref as S


# ------------------------------------------------------------------ the dispatch
def regime(page_size, kbn):
    return "<" if page_size < kbn else ("=" if page_size == kbn else ">")


def path(B, H, Hkv, Nq, page_size, max_pages, D, causal, splits):
    """(path key, launches) of one call; splits = 0 resolves from the padded shape as the library does."""
    if page_size < 16 or page_size & (page_size - 1):
        raise ValueError(f"not a supported page size: {page_size}")
    key, launches = S.path(B, H, Hkv, Nq, max_pages * page_size, D, causal, splits)
    return key + (regime(page_size, key[1]),), launches


def instantiation(key):
    return key[:5]


def reachable():
    """Every path key: the seqlens paths (three kernel families, causal or not, one split or two, short or long query
    heads) in every page-size regime."""
    keys = set()
    for D in (40, 128, 264):
        kbn, _ = M.kernel_shape(D)
        for ps in (16, kbn, 2 * kbn):
            for causal in (False, True):
                for splits in (1, 2):
                    for Nq in (1, 256):
                        keys.add(path(1, 4, 2, Nq, ps, 4096 // ps, D, causal, splits)[0])
    return keys


_MANGLED = re.compile(r"attn_fwd_paged_kernelILi(\d+)ELi(\d+)ELi(\d+)ELb([01])ELb([01])E")
_DEMANGLED = re.compile(r"attn_fwd_paged_kernel<(\d+), (\d+), (\d+), (true|false), (true|false)>")


def parse_instantiations(names):
    out = []
    for name in names:
        for m in list(_MANGLED.finditer(name)) + list(_DEMANGLED.finditer(name)):
            a = m.groups()
            out.append((int(a[0]), int(a[1]), int(a[2]), *(x in ("1", "true") for x in a[3:])))
    return out


# ------------------------------------------------------------------ the kernel's sub-loads and the gather
def sub_loads(j, kbn, page_size, lk, table_row):
    """[(byte offset in the ring slot, first pool row, table index read)] of the kBN / R sub-loads of key block j of a
    sequence with lk >= 1 keys (attn_sm90.cuh, kPaged): R = min(page_size, kBN) rows each; sub-loads past the last
    used page read that page again, so no table index >= ceil(lk / page_size) is read."""
    R_ = min(page_size, kbn)
    last = -(-lk // page_size) - 1
    out = []
    for i in range(kbn // R_):
        t = j * kbn + i * R_
        pi = min(t // page_size, last)
        out.append((i * R_ * 128, int(table_row[pi]) * page_size + t % page_size, pi))
    return out


def gather(pool, table, lk, Nk):
    """The contiguous padded cache [B,Hkv,Nk,D] of pool [num_pages, page_size, Hkv, D] (torch) through table [B, max_pages]
    (rows >= lk[b] zero): what a caller without the paged entry builds before every call."""
    import torch
    num_pages, ps, Hkv, D = pool.shape
    B = table.shape[0]
    out = torch.zeros(B, Hkv, Nk, D, dtype=pool.dtype, device=pool.device)
    for b in range(B):
        n = -(-lk[b] // ps)
        if n == 0:
            continue
        rows = pool[table[b, :n].long()].reshape(n * ps, Hkv, D)[:lk[b]]
        out[b, :, :lk[b]] = rows.transpose(0, 1)
    return out


# ------------------------------------------------------------------ the GPU case table
# One row per path key.  Each row's sequences have the key lengths 0, 1, kBN - 1, kBN + 1, page_size - 1,
# page_size + 1 and the full padded Nk, and query lengths that mix 0 or 1 with full ones; causal rows include Lq > Lk.
# Shapes: D = 40 / 64 (kDS 64, kBN 128), 72 / 128 (kDS 128, kBN 64), 136 / 264 and 520 / 776 / 1000 (kDS 256; three
# and four slabs, from 776 on a K/V ring shorter than one key block); G in {1, 4, 8}; Nq = 1 / 5 (decoding, packed
# tiles) and 130 (per-head tiles when causal).
Case = namedtuple("Case", "H Hkv Nq page_size max_pages D causal splits lq lk gens")

_FAMILIES = [   # (head dims, kBN, page sizes below / at / above kBN with the table width that gives Nk ~ 800)
    ((40, 64), 128, ((16, 50), (128, 6), (256, 3))),
    ((72, 128), 64, ((16, 50), (64, 12), (256, 3))),
    ((136, 264), 64, ((32, 25), (64, 12), (128, 6))),
    ((520, 776, 1000), 64, ((16, 50), (64, 12), (256, 3))),   # a K/V ring shorter than one block (attn_ring_ref)
]
# (causal, split, Nq): the six seqlens paths of a family (non-causal rows are packed whatever Nq)
_PATHS = [(False, False, 1), (False, True, 130), (True, False, 5), (True, False, 130), (True, True, 5),
          (True, True, 130)]
_LQ = {1: (1, 1, 0, 1, 1, 1, 1), 5: (5, 1, 0, 5, 5, 2, 5), 130: (130, 1, 5, 0, 130, 77, 129)}
_HEADS = [(4, 4), (8, 2), (8, 1)]
_ADVERSARIAL = [g for g in R.GENERATORS if g != "randn"]


def _lk(kbn, ps, nk):
    return (0, 1, kbn - 1, kbn + 1, ps - 1, ps + 1, nk)


def _rows():
    rows, n = [], 0
    for Ds, kbn, pages in _FAMILIES:
        for ps, maxp in pages:
            for causal, split, Nq in _PATHS:
                H, Hkv = _HEADS[n % 3]
                gens = ("randn", (M.PROBES if causal else _ADVERSARIAL)[n % (2 if causal else 5)])
                rows.append(Case(H, Hkv, Nq, ps, maxp, Ds[n % len(Ds)], causal, 2 + n % 5 if split else 1, _LQ[Nq],
                                 _lk(kbn, ps, ps * maxp), gens))
                n += 1
    return rows


CASES_BY_SHAPE = _rows()
CASES = [(c, gen) for c in CASES_BY_SHAPE for gen in c.gens]


def case_key(c):
    return path(len(c.lq), c.H, c.Hkv, c.Nq, c.page_size, c.max_pages, c.D, c.causal, c.splits)[0]


def cases_by_key(cases=None):
    out = {}
    for c, gen in (CASES if cases is None else cases):
        out.setdefault(case_key(c), []).append((c, gen))
    return out
