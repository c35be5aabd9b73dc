"""Per-sequence lengths (b200_fmha_fwd_f16_seqlens): the fp64 reference, the dispatch and the kernel's key ranges
restated on the CPU, and the GPU case table.  Used by test_attn_seqlens_coverage.py, test_attn_seqlens_sharpness.py
and test_attn_seqlens_gpu.py.

Semantics.  q, o [B,H,Nq,D] and k, v [B,Hkv,Nk,D] are padded; sequence b has Lq_b = clamp(seqlens_q[b], 0, Nq) queries
and Lk_b = clamp(seqlens_k[b], 0, Nk) keys.  Query i of sequence b sees key j when i < Lq_b, j < Lk_b and, with the
mask, j <= i + (Lk_b - Lq_b).  Rows that see no key (padded rows included) are O = 0, lse = -inf exactly.

A path key is (kDS, kBN, kWG, kCausal, kSplit, tiling): the first five are the template arguments of
attn_fwd_seqlens_kernel, tiling is "per-head" (causal with Nq >= the tile rows: every query head has tiles of its own)
or "packed" (tiles cut across the packed rows of a K/V group; always without the mask).
"""
from __future__ import annotations

import re
from collections import namedtuple

import numpy as np

import attn_mask_ref as M
import attn_paths as P
import attn_ref as R
import attn_split_ref as SR


def clamp(lens, n):
    return [min(max(int(x), 0), n) for x in lens]


# ------------------------------------------------------------------ the dispatch
def path(B, H, Hkv, Nq, Nk, D, causal, splits):
    """(path key, launches) of one call; splits = 0 resolves from the padded shape as the library does."""
    if D % 8 or D > 1024 or H % Hkv:
        raise ValueError(f"not a supported call: H{H} Hkv{Hkv} D{D}")
    if splits == 0:
        from leetcuda_b200 import _capi
        splits = _capi.lib().b200_fmha_fwd_f16_gqa_splits(B, H, Hkv, Nq, Nk, D)
    kbn, rows = M.kernel_shape(D)
    ds = P._SLAB[R.family(D)[0]]
    tiling = "per-head" if causal and Nq >= rows else "packed"
    return (ds, kbn, rows // 64, bool(causal), splits > 1, tiling), 1 + (splits > 1)


def instantiation(key):
    return key[:5]


def reachable():
    """Every path key: the three kernel families, causal or not, one split or two, short or long query heads."""
    keys = set()
    for D in (40, 128, 264):
        for causal in (False, True):
            for splits in (1, 2):
                for Nq in (1, 256):
                    keys.add(path(1, 4, 2, Nq, 512, D, causal, splits)[0])
    return keys


_MANGLED = re.compile(r"attn_fwd_seqlens_kernelILi(\d+)ELi(\d+)ELi(\d+)ELb([01])ELb([01])E")
_DEMANGLED = re.compile(r"attn_fwd_seqlens_kernel<(\d+), (\d+), (\d+), (true|false), (true|false)>")


def parse_instantiations(names):
    out = []
    for name in names:
        for m in list(_MANGLED.finditer(name)) + list(_DEMANGLED.finditer(name)):
            a = m.groups()
            out.append((int(a[0]), int(a[1]), int(a[2]), *(x in ("1", "true") for x in a[3:])))
    return out


# ------------------------------------------------------------------ the kernel's key ranges
def tile_nkv(first, end, lq, lk, Nq, kbn, causal, diag_padded=None, short=0):
    """Key blocks a CTA whose query positions are [first, end) visits (attn_sm90.cuh kv_blocks, kSeqlens).  Mutations:
    diag_padded = (Nq, Nk) takes the diagonal from the padded shape; short = 1 visits one block fewer."""
    num_kv = -(-lk // kbn)
    end = min(end, lq)
    if end <= first:
        return 0
    if not causal:
        return max(num_kv - short, 0)
    diag = lk - lq if diag_padded is None else diag_padded[1] - diag_padded[0]
    keys = end + diag
    return 0 if keys <= 0 else max(min(num_kv, -(-keys // kbn)) - short, 0)


def tiles(G, Nq, D, causal, lq, lk, **mut):
    """[(packed rows of the CTA, nkv)] over the G*Nq packed rows of a K/V head of one sequence."""
    kbn, per = M.kernel_shape(D)
    rows = G * Nq
    out = []
    if causal and Nq >= per:
        for g in range(G):
            for t0 in range(0, Nq, per):
                end = min(t0 + per, Nq)
                out.append((np.arange(g * Nq + t0, g * Nq + end), tile_nkv(t0, end, lq, lk, Nq, kbn, causal, **mut)))
        return out
    for q0 in range(0, rows, per):
        last = min(q0 + per, rows) - 1
        cross = last // Nq != q0 // Nq
        first, end = (0, Nq) if cross else (q0 % Nq, last % Nq + 1)
        out.append((np.arange(q0, last + 1), tile_nkv(first, end, lq, lk, Nq, kbn, causal, **mut)))
    return out


def visible(Nq, Nk, lq, lk, causal):
    """[Nq, Nk] bool: the keys query i of a sequence with lq queries and lk keys sees."""
    i, j = np.arange(Nq)[:, None], np.arange(Nk)[None, :]
    vis = (i < lq) & (j < lk)
    return vis & (j <= i + (lk - lq)) if causal else vis


def part_masks(G, Nq, Nk, D, causal, splits, lq, lk):
    """[S, G*Nq, Nk] bool: key j is in split z of packed row r and visible to it (one sequence)."""
    kbn, _ = M.kernel_shape(D)
    out = np.zeros((splits, G * Nq, Nk), bool)
    for r, nkv in tiles(G, Nq, D, causal, lq, lk):
        for z, (b, e) in enumerate(SR.split_ranges(nkv, splits)):
            out[z, r, b * kbn:min(e * kbn, Nk)] = True
    return out & np.tile(visible(Nq, Nk, lq, lk, causal), (G, 1))[None]


# ------------------------------------------------------------------ fp64 references
def reference(q, k, v, scale, causal, lq, lk, exact_scores=False):
    """attn_split_ref.masked_reference with every sequence's visibility (q [B,H,Nq,D], k, v [B,Hkv,Nk,D] torch)."""
    import torch
    B, H, Nq, _ = q.shape
    Nk = k.shape[2]
    G = H // k.shape[1]
    vis = np.stack([visible(Nq, Nk, lq[b], lk[b], causal) for b in range(B)])[:, None]
    vis = torch.from_numpy(vis).to(q.device)
    return SR.masked_reference(q, SR.expand(k, G), SR.expand(v, G), scale, vis, exact_scores)


def part_references(q, k, v, scale, causal, splits, lq, lk, exact_scores=False):
    """fp64 references of the S parts of every row, as attn_split_ref.part_references, per sequence."""
    import torch
    B, H, Nq, D = q.shape
    G = H // k.shape[1]
    Nk = k.shape[2]
    masks = np.stack([SR.head_masks(part_masks(G, Nq, Nk, D, causal, splits, lq[b], lk[b]), H, G, Nq)
                      for b in range(B)], axis=1)                 # [S, B, H, Nq, Nk]
    masks = torch.from_numpy(masks).to(q.device)
    ke, ve = SR.expand(k, G), SR.expand(v, G)
    return [SR.masked_reference(q, ke, ve, scale, masks[z], exact_scores) for z in range(splits)]


# ------------------------------------------------------------------ the GPU case table
# Every row mixes the lengths of its sequences: Lk 0, 1, kBN - 1, kBN, kBN + 1, ragged and Nk; Lq 0, 1, 5 and Nq;
# causal rows with Lq > Lk.  Shapes: D = 40 / 64 (kDS 64, kBN 128), 72 / 128 (kDS 128, kBN 64), 136 / 264 (kDS 256),
# and 520 / 776 / 1000 (kDS 256: three slabs, the last one 8 columns, and four; from 776 on the K/V ring holds less
# than one key block, at 1000 it is at its smallest); G in {1, 4, H}; Nq = 1 / 5 (decoding, packed tiles) and 130
# (per-head tiles with Nq >= 128 rows, and Nq >= 64).
Case = namedtuple("Case", "H Hkv Nq Nk D causal splits lq lk gens")
F, T = False, True
_LK128 = (0, 1, 127, 128, 129, 300, 777)
_LK64 = (0, 1, 63, 64, 65, 300, 777)

CASES_BY_SHAPE = [
    Case(4, 4, 1, 777, 40, F, 1, (1, 0, 1, 1, 1, 1, 1), _LK128, ("randn", "neg_scores")),
    Case(8, 2, 5, 777, 64, T, 1, (5, 1, 0, 5, 5, 2, 5), _LK128, ("randn", "tail_max", "diag_gather")),
    Case(8, 2, 130, 777, 40, T, 1, (130, 1, 5, 0, 130, 77, 129), _LK128, ("randn", "front_max", "future_max")),
    Case(8, 8, 130, 300, 64, F, 1, (130, 5, 1, 0, 130, 64, 100), (0, 1, 127, 128, 129, 250, 300), ("randn", "one_hot")),
    Case(8, 1, 1, 777, 40, F, 3, (1, 1, 0, 1, 1, 1, 1), _LK128, ("randn", "ramp_max")),
    Case(4, 2, 130, 777, 64, T, 4, (130, 5, 1, 130, 0, 3, 100), _LK128, ("randn", "neg_scores", "future_max")),
    Case(4, 4, 5, 777, 40, T, 2, (5, 5, 1, 0, 5, 5, 5), _LK128, ("randn", "tail_max", "diag_gather")),
    Case(8, 8, 130, 777, 64, F, 2, (130, 1, 0, 5, 130, 130, 17), _LK128, ("randn", "front_max")),
    Case(4, 4, 1, 777, 128, F, 1, (1, 1, 1, 0, 1, 1, 1), _LK64, ("randn", "ramp_max")),
    Case(8, 2, 5, 777, 72, T, 1, (5, 1, 5, 5, 0, 4, 5), _LK64, ("randn", "one_hot", "diag_gather")),
    Case(8, 2, 130, 777, 128, T, 1, (130, 1, 5, 130, 0, 90, 129), _LK64, ("randn", "neg_scores", "future_max")),
    Case(8, 8, 130, 300, 72, F, 1, (130, 0, 1, 5, 130, 64, 100), (0, 1, 63, 64, 65, 250, 300), ("randn", "tail_max")),
    Case(8, 1, 1, 777, 128, F, 6, (1, 1, 0, 1, 1, 1, 1), _LK64, ("randn", "front_max")),
    Case(4, 2, 130, 777, 72, T, 3, (130, 5, 0, 1, 130, 7, 64), _LK64, ("randn", "one_hot", "future_max")),
    Case(8, 8, 5, 777, 128, T, 4, (5, 0, 1, 5, 5, 5, 5), _LK64, ("randn", "ramp_max", "diag_gather")),
    Case(8, 8, 130, 777, 72, F, 2, (130, 1, 0, 5, 130, 33, 99), _LK64, ("randn", "neg_scores")),
    Case(4, 4, 1, 777, 136, F, 1, (1, 1, 0, 1, 1, 1, 1), _LK64, ("randn", "tail_max")),
    Case(8, 2, 5, 300, 264, T, 1, (5, 1, 5, 0, 5, 3, 5), (0, 1, 63, 64, 65, 200, 300), ("randn", "front_max",
                                                                                          "diag_gather")),
    Case(8, 2, 130, 777, 136, T, 1, (130, 1, 5, 130, 0, 64, 129), _LK64, ("randn", "ramp_max", "future_max")),
    Case(4, 4, 130, 300, 264, F, 1, (130, 5, 1, 0, 130, 64, 100), (0, 1, 63, 64, 65, 250, 300), ("randn", "one_hot")),
    Case(8, 1, 1, 777, 136, F, 5, (1, 1, 1, 0, 1, 1, 1), _LK64, ("randn", "neg_scores")),
    Case(4, 2, 130, 777, 136, T, 2, (130, 5, 1, 0, 130, 9, 64), _LK64, ("randn", "tail_max", "future_max")),
    Case(8, 8, 5, 777, 264, T, 3, (5, 0, 1, 5, 5, 5, 5), _LK64, ("randn", "front_max", "diag_gather")),
    Case(8, 8, 130, 300, 136, F, 3, (130, 1, 0, 5, 130, 70, 99), (0, 1, 63, 64, 65, 250, 300), ("randn", "one_hot")),
    # head dims 520 / 776 / 1000: three slabs and four, a K/V ring shorter than one key block (attn_ring_ref)
    Case(4, 4, 1, 777, 520, F, 1, (1, 1, 0, 1, 1, 1, 1), _LK64, ("randn", "tail_max")),
    Case(8, 2, 5, 777, 776, T, 1, (5, 1, 5, 5, 0, 4, 5), _LK64, ("randn", "front_max", "diag_gather")),
    Case(8, 2, 130, 777, 1000, T, 1, (130, 1, 5, 130, 0, 90, 129), _LK64, ("randn", "ramp_max", "future_max")),
    Case(8, 1, 1, 777, 1000, F, 5, (1, 1, 1, 0, 1, 1, 1), _LK64, ("randn", "one_hot")),
    Case(4, 2, 130, 777, 776, T, 2, (130, 5, 1, 0, 130, 9, 64), _LK64, ("randn", "neg_scores", "future_max")),
    Case(8, 8, 5, 777, 520, T, 3, (5, 0, 1, 5, 5, 5, 5), _LK64, ("randn", "tail_max", "diag_gather")),
]

CASES = [(c, gen) for c in CASES_BY_SHAPE for gen in c.gens]


def case_key(c):
    return path(len(c.lq), c.H, c.Hkv, c.Nq, c.Nk, c.D, c.causal, c.splits)[0]


def cases_by_key(cases=None):
    out = {}
    for c, gen in (CASES if cases is None else cases):
        out.setdefault(case_key(c), []).append((c, gen))
    return out
