"""The K/V ring of the D > 128 attention kernels (csrc/attn_capi.cu fmha_dispatch, csrc/attn_sm90.cuh) restated on the
CPU, and the regimes a case of the GPU tables reaches in it.  Used by test_attn_ring_coverage.py (CPU gate) and
test_attn_ring_smem_gpu.py (the restated shared memory against the launches the profiler records).

The ring.  Q (all of D, ceil(D/64) chunks of 8 KiB per consumer warpgroup) stays in shared memory; K and V stream
through `ring` slots next to it, as many as fit in 227 KiB, at most 16 (attn_capi.cu fmha_dispatch, the lines after
"ring: every slot that fits next to Q"):
    fixed = smem_bytes(wgs, slot, nq, 0)
    ring  = min(16, (227 KiB - fixed) / (slot + 16 + stage))
    smem  = smem_bytes(wgs, slot, nq, ring) + ring stage
where attn_sm90.cuh's smem_bytes(wgs, slot, nq, ring) = wgs nq 8192 + ring slot + 8 (1 + 2 ring) + wgs 256 + 1024,
slot = 128 kBN bytes (natural V) and, for fp8 K/V, stage = 64 kBN + 8: every slot has an e4m3 staging chunk and a
third barrier.  The kernels declare no static shared memory, so smem is what a launch takes.

A key block of one CTA takes nq = ceil(D/64) K chunks and its slab's V chunks, min(kDS/64, ceil((D - slab kDS)/64)) of
them, in ring order.  When a block takes more chunks than the ring holds ("wrap"), the producer refills slots of the
block the consumers are still reading: for fp16 / bf16 from D = 776 (ring 15 < 17), for fp8 K/V from D = 528 (ring
12 < 13).  The ring is at its smallest, 12 slots, for D > 960 (fp8: 8 slots for D > 896).

Regimes.  regimes(kind, T, case) names what a case of the tables runs in this ring: three slabs whose last one has a
single V chunk, four slabs, a ring shorter than one key block, the kind's smallest ring, and in a ring that wraps: the
causal mask, a split, the partial last key block whose V rows warp 1 zeroes (fp8: the converters) below the padded Nk,
and paged sub-loads of 16-key pages or of pages larger than kBN.
"""
from __future__ import annotations

import attn_bf16_ref as BF
import attn_fp8kv_ref as F
import attn_paged_ref as P
import attn_paths as AP
import attn_seqlens_ref as S

MAX_SMEM = 227 * 1024     # attn_capi.cu: kMaxSmem
MAX_RING = 16             # attn_capi.cu: "if (p.ring > 16) p.ring = 16"

THREE_SLABS = "three slabs, the last one a single V chunk"
FOUR_SLABS = "four slabs"
WRAP = "ring shorter than one key block"
SMALLEST = "the smallest ring"
WRAP_CAUSAL = "wrap with the causal mask"
WRAP_SPLIT = "wrap with a split"
WRAP_PARTIAL = "wrap with a partial last key block below the padded Nk"
WRAP_PAGE16 = "wrap with 16-key pages"
WRAP_BIG_PAGE = "wrap with pages larger than kBN"

# (kind, T): the attention kernels of head dims > 128 and their element types.  "dense" is attn_fwd_kernel<256, 64, 1,
# ...> (fp16 only); "seqlens" and "paged" the per-sequence-length and paged kernels, with fp16 or bf16 elements or with
# e4m3 K/V and half or bf16 Q/O.
KINDS = [("dense", "half")] + [(k, t) for k in ("seqlens", "paged") for t in ("half", "bf16", "fp8-half", "fp8-bf16")]


def required(kind):
    """The regimes the tables must reach for a kernel kind."""
    out = [THREE_SLABS, FOUR_SLABS, WRAP, SMALLEST, WRAP_CAUSAL, WRAP_SPLIT]
    if kind != "dense":
        out.append(WRAP_PARTIAL)   # the dense kernel reads zeros past Nk from TMA and zeroes nothing
    if kind == "paged":
        out += [WRAP_PAGE16, WRAP_BIG_PAGE]
    return out


# ------------------------------------------------------------------ the ring, as fmha_dispatch sizes it
def family(D):
    """(kDS, kBN, consumer warpgroups): attn_capi.cu family()."""
    ds = 64 if D <= 64 else (128 if D <= 128 else 256)
    return ds, (128 if ds == 64 else 64), (1 if ds == 256 else 2)


def nq(D):
    return -(-D // 64)


def slabs(D):
    return -(-D // family(D)[0])


def chunks_per_block(D, slab):
    """Ring slots one key block of slab `slab` takes: its nq K chunks, then the slab's V chunks (attn_sm90.cuh, nvc)."""
    ds = family(D)[0]
    return nq(D) + min(ds // 64, -(-(D - slab * ds) // 64))


def _slot(D):
    return 128 * family(D)[1]   # attn_sm90.cuh slot_bytes, natural V


def _stage(D, fp8):
    return 64 * family(D)[1] + 8 if fp8 else 0


def _smem(D, ring):
    """attn_sm90.cuh smem_bytes(wgs, slot, nq, ring)."""
    wgs = family(D)[2]
    return wgs * nq(D) * 8192 + ring * _slot(D) + 8 * (1 + 2 * ring) + wgs * 64 * 4 + 1024


def ring(D, fp8=False):
    """K/V ring slots of head dim D (attn_capi.cu fmha_dispatch)."""
    r = min(MAX_RING, (MAX_SMEM - _smem(D, 0)) // (_slot(D) + 16 + _stage(D, fp8)))
    if r < 2:
        raise ValueError(f"D{D}: no ring fits")
    return r


def smem_bytes(D, fp8=False):
    """Dynamic shared memory of the launch (fmha_dispatch's smem)."""
    r = ring(D, fp8)
    return _smem(D, r) + r * _stage(D, fp8)


def smallest_ring(fp8):
    return min(ring(D, fp8) for D in range(136, 1025, 16 if fp8 else 8))


# ------------------------------------------------------------------ the regimes of a case
def _lengths(kind, case):
    """(padded Nk, [(Lq_b, Lk_b)]) of a case; a dense case (no lengths) has B sequences of Nq queries and Nk keys."""
    if kind == "paged":
        nk = case.page_size * case.max_pages
    else:
        nk = case.Nk
    if not hasattr(case, "lk"):
        return nk, [(case.Nq, nk)] * getattr(case, "B", 2)
    return nk, [(min(max(a, 0), case.Nq), min(max(b, 0), nk)) for a, b in zip(case.lq, case.lk)]


def regimes(kind, T, case):
    """The regimes a case reaches: kind "dense" (attn_paths.Case, D > 128 only), "seqlens" (attn_seqlens_ref.Case or
    attn_bf16_ref.Dense, which runs the seqlens kernel) or "paged"; T "half", "bf16", "fp8-half" or "fp8-bf16"."""
    D = case.D
    if D <= 128:   # one slab, a ring of several key blocks
        return set()
    fp8 = T.startswith("fp8")
    r = ring(D, fp8)
    n = slabs(D)
    out = set()
    if n == 3 and chunks_per_block(D, 2) - nq(D) == 1:
        out.add(THREE_SLABS)
    if n == 4:
        out.add(FOUR_SLABS)
    if r == smallest_ring(fp8):
        out.add(SMALLEST)
    if r >= max(chunks_per_block(D, s) for s in range(n)):
        return out
    out.add(WRAP)
    if case.causal:
        out.add(WRAP_CAUSAL)
    if case.splits > 1:
        out.add(WRAP_SPLIT)
    kbn = family(D)[1]
    if kind != "dense":
        nk, seqs = _lengths(kind, case)
        # attn_sm90.cuh vz: the partial block of a sequence with a query; paged: any partial block
        if any(lq > 0 and lk % kbn and (kind == "paged" or lk < nk) for lq, lk in seqs):
            out.add(WRAP_PARTIAL)
    if kind == "paged":
        if case.page_size == 16:
            out.add(WRAP_PAGE16)
        if case.page_size > kbn:
            out.add(WRAP_BIG_PAGE)
    return out


def table_rows():
    """[(kind, T, case)] of every case table that runs a D > 128 attention kernel: attn_paths (dense fp16),
    attn_seqlens_ref, attn_paged_ref, attn_bf16_ref (its dense rows run the seqlens kernel) and attn_fp8kv_ref."""
    rows = [("dense", "half", c) for c in AP.CASES_BY_SHAPE]
    rows += [("seqlens", "half", c) for c in S.CASES_BY_SHAPE] + [("paged", "half", c) for c in P.CASES_BY_SHAPE]
    rows += [("paged" if k == "paged" else "seqlens", "bf16", c) for k, c in BF.CASES]
    rows += [("paged" if k == "paged" else "seqlens", "fp8-" + t, c) for t, k, c in F.CASES]
    return rows


def missing(rows):
    """{(kind, T, regime)} the rows do not reach."""
    got = {(kind, T, g) for kind, T, c in rows for g in regimes(kind, T, c)}
    return {(kind, T, g) for kind, T in KINDS for g in required(kind)} - got
