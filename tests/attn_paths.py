"""The attention dispatch (csrc/attn_capi.cu: fmha_impl, fmha_dispatch, launch_attn) restated on the CPU, the set of
paths it can reach, and the GPU case table that runs each of them.  Used by test_attn_path_coverage.py (CPU gate) and
test_attn_paths_gpu.py.

A path key is (kDS, kBN, kWG, kVT, kCausal, kGQA, kSplit, prepass, rms, tiling):
  * the first seven are the template arguments of attn_fwd_kernel;
  * prepass: V^T [B,Hkv,D,Nk] with D > 128 goes through transpose_dn_to_nd_kernel first, and the kernel reads natural V;
  * rms: "-", "row" (fused RMS norm inside one CTA) or "cluster" (the slabs of a query tile form a cluster);
  * tiling: for the kCausal && kGQA kernels, "per-head" (p.tph > 0: every query head has tiles of its own) or "packed"
    (tiles cut across the packed rows of a K/V group); "-" for every other kernel, which ignores p.tph.
"""
from __future__ import annotations

import re
from collections import namedtuple

import attn_mask_ref as M
import attn_ref as R

_SLAB = {"D<=64": 64, "64<D<=128": 128, "D>128": 256}   # columns of O per CTA, by attn_ref.family


def rms_supported(D):
    return D <= 256 or D in (384, 512)


def path(B, H, Hkv, Nq, Nk, D, vt, causal, splits, rms):
    """(path key, launches) of one call.  splits = 0 is resolved the way the library resolves it
    (b200_fmha_fwd_f16_gqa_splits); rms: through b200_fmha_fwd_f16_rmsnorm (non-causal, Nq = Nk, G = 1, no split)."""
    if D % 8 or D > 1024 or H % Hkv or (vt and Nk % 8):
        raise ValueError(f"not a supported call: H{H} Hkv{Hkv} Nk{Nk} D{D} vt={vt}")
    G = H // Hkv
    if rms and (causal or Nq != Nk or G != 1 or splits != 1 or not rms_supported(D)):
        raise ValueError("the fused RMS norm is non-causal with Nq = Nk, G = 1, one split and D <= 256 or 384, 512")
    if splits == 0:
        from leetcuda_b200 import _capi
        splits = _capi.lib().b200_fmha_fwd_f16_gqa_splits(B, H, Hkv, Nq, Nk, D)
    split = splits > 1
    kbn, rows = M.kernel_shape(D)
    ds = _SLAB[R.family(D)[0]]
    prepass = bool(vt) and D > 128          # fmha_impl restores the natural layout, the kernel sees vt = False
    kvt = bool(vt) and not prepass
    # launch_attn: a split runs <.., causal, causal, true> for every G; unsplit causal runs kGQA when G > 1
    kgqa = causal and (split or G > 1)
    tiling = "-" if not (causal and kgqa) else ("per-head" if Nq >= rows else "packed")
    slabs = -(-D // ds)
    key = (ds, kbn, rows // 64, kvt, bool(causal), kgqa, split, prepass,
           "-" if not rms else ("cluster" if slabs > 1 else "row"), tiling)
    return key, 1 + prepass + split


def instantiation(key):
    return key[:7]


def reachable():
    """Every path key the library can take: D = 8 .. 1024, both V layouts, causal or not, G = 1 or 2, one split or two,
    Nq below or at least the tile rows, and the fused RMS norm where it exists."""
    keys = set()
    for D in range(8, 1025, 8):
        for vt in (False, True):
            for causal in (False, True):
                for Hkv in (2, 1):              # H = 2: G = 1 or 2
                    for splits in (1, 2):
                        for Nq in (8, 256):
                            keys.add(path(1, 2, Hkv, Nq, 256, D, vt, causal, splits, False)[0])
        if rms_supported(D):
            for vt in (False, True):
                keys.add(path(1, 2, 2, 256, 256, D, vt, False, 1, True)[0])
    return keys


# ------------------------------------------------------------------ attn_fwd_kernel<...> in symbol names
_MANGLED = re.compile(r"attn_fwd_kernelILi(\d+)ELi(\d+)ELi(\d+)ELb([01])ELb([01])ELb([01])ELb([01])E")
_DEMANGLED = re.compile(r"attn_fwd_kernel<(\d+), (\d+), (\d+), (true|false), (true|false), (true|false), "
                        r"(true|false)>")


def parse_instantiations(names):
    """The attn_fwd_kernel template arguments in the given symbol names, mangled or demangled."""
    out = []
    for name in names:
        for m in list(_MANGLED.finditer(name)) + list(_DEMANGLED.finditer(name)):
            a = m.groups()
            out.append((int(a[0]), int(a[1]), int(a[2]), *(x in ("1", "true") for x in a[3:])))
    return out


# ------------------------------------------------------------------ the GPU case table
# One row per shape; every generator of the row is one case (attn_ref / attn_mask_ref generators).  The shapes reach
# the edges of their kernel:
#   D = 40 (a ragged 64-column slab), 72 (ragged 128), 136 (one ragged 256-column slab), 256 (one full slab), 264 (two
#   slabs, the second 8 columns wide), 384 / 512 (the RMS cluster), 520 (three slabs, the last 8 columns wide), 776 /
#   1000 (four slabs; the K/V ring holds less than one key block, at 1000 it is at its smallest: attn_ring_ref);
#   Nk = 776 = 12 * 64 + 8 with V^T (Nk % 8 == 0 there): the last V^T box is 56 keys out of bounds, 777 / 300 / 1000
#   ragged otherwise;
#   Nq = 1 and 5 (packed decoding, speculative decoding), 130 (>= the tile rows: per-head tiles, a ragged last tile);
#   G in {1, 4, H} for the splits; split counts above the key blocks of a CTA (9 > 776 / 128, 17 > 1000 / 64, and the
#   short causal tiles of 130 rows) leave some splits empty.
Case = namedtuple("Case", "B H Hkv Nq Nk D vt causal splits rms gens")
F, T = False, True
_A = ("neg_scores", "front_max", "tail_max", "ramp_max", "one_hot")   # adversarial generators, taken in turn

CASES_BY_SHAPE = [
    # D <= 64 (kDS 64, kBN 128), natural V
    Case(2, 4, 2, 130, 777, 40, F, F, 1, F, ("randn", "neg_scores")),
    Case(1, 2, 2, 130, 776, 64, F, T, 1, F, ("randn", "tail_max", "diag_gather")),
    Case(1, 8, 2, 130, 777, 40, F, T, 1, F, ("randn", "front_max", "future_max")),
    Case(2, 8, 2, 5, 300, 64, F, T, 1, F, ("randn", "ramp_max", "diag_gather")),
    Case(1, 8, 1, 1, 1000, 40, F, F, 9, F, ("randn", "one_hot")),
    Case(1, 8, 2, 130, 777, 64, F, T, 7, F, ("randn", "neg_scores", "future_max")),
    Case(2, 8, 8, 5, 777, 40, F, T, 3, F, ("randn", "tail_max", "diag_gather")),
    Case(1, 2, 2, 130, 130, 64, F, F, 1, T, ("randn", "one_hot")),
    # D <= 64, transposed V (the vt kernel)
    Case(2, 4, 2, 130, 776, 64, T, F, 1, F, ("randn", "front_max")),
    Case(1, 2, 2, 130, 776, 40, T, T, 1, F, ("randn", "ramp_max", "future_max")),
    Case(1, 8, 2, 130, 776, 64, T, T, 1, F, ("randn", "one_hot", "diag_gather")),
    Case(2, 8, 2, 5, 776, 40, T, T, 1, F, ("randn", "neg_scores", "future_max")),
    Case(1, 8, 8, 5, 776, 64, T, F, 9, F, ("randn", "tail_max")),
    Case(2, 4, 1, 1, 776, 40, T, F, 4, F, ("randn", "ramp_max")),
    Case(1, 8, 2, 130, 776, 40, T, T, 9, F, ("randn", "front_max", "diag_gather")),
    Case(1, 8, 1, 5, 776, 64, T, T, 5, F, ("randn", "one_hot", "future_max")),
    Case(1, 2, 2, 136, 136, 40, T, F, 1, T, ("randn", "neg_scores")),
    # 64 < D <= 128 (kDS 128, kBN 64), natural V
    Case(2, 4, 2, 130, 777, 72, F, F, 1, F, ("randn", "tail_max")),
    Case(1, 2, 2, 130, 1000, 128, F, T, 1, F, ("randn", "ramp_max", "diag_gather")),
    Case(1, 8, 2, 130, 777, 72, F, T, 1, F, ("randn", "one_hot", "future_max")),
    Case(2, 8, 2, 5, 777, 128, F, T, 1, F, ("randn", "neg_scores", "diag_gather")),
    Case(1, 8, 8, 1, 1000, 128, F, F, 17, F, ("randn", "front_max")),
    Case(1, 4, 4, 130, 300, 72, F, T, 6, F, ("randn", "tail_max", "future_max")),
    Case(2, 8, 1, 5, 777, 128, F, T, 4, F, ("randn", "ramp_max", "diag_gather")),
    Case(1, 2, 2, 129, 129, 72, F, F, 1, T, ("randn", "front_max")),
    # 64 < D <= 128, transposed V
    Case(2, 4, 2, 130, 776, 128, T, F, 1, F, ("randn", "one_hot")),
    Case(1, 2, 2, 130, 776, 72, T, T, 1, F, ("randn", "neg_scores", "future_max")),
    Case(1, 8, 2, 130, 776, 128, T, T, 1, F, ("randn", "tail_max", "diag_gather")),
    Case(2, 8, 2, 5, 776, 72, T, T, 1, F, ("randn", "front_max", "future_max")),
    Case(1, 8, 2, 5, 776, 72, T, F, 17, F, ("randn", "ramp_max")),
    Case(1, 8, 8, 130, 776, 128, T, T, 7, F, ("randn", "one_hot", "diag_gather")),
    Case(1, 8, 1, 1, 776, 128, T, T, 3, F, ("randn", "neg_scores", "future_max")),
    Case(1, 2, 2, 136, 136, 128, T, F, 1, T, ("randn", "tail_max")),
    # D > 128 (kDS 256, kBN 64, one consumer warpgroup), natural V
    Case(2, 4, 2, 130, 777, 136, F, F, 1, F, ("randn", "ramp_max")),
    Case(1, 2, 2, 130, 300, 264, F, T, 1, F, ("randn", "one_hot", "diag_gather")),
    Case(1, 8, 2, 130, 777, 136, F, T, 1, F, ("randn", "neg_scores", "future_max")),
    Case(2, 8, 2, 5, 300, 264, F, T, 1, F, ("randn", "front_max", "diag_gather")),
    Case(1, 4, 1, 1, 1000, 136, F, F, 17, F, ("randn", "tail_max")),
    Case(1, 8, 8, 130, 777, 264, F, T, 5, F, ("randn", "ramp_max", "future_max")),
    Case(2, 8, 2, 5, 777, 136, F, T, 2, F, ("randn", "one_hot", "diag_gather")),
    Case(1, 2, 2, 130, 130, 256, F, F, 1, T, ("randn", "neg_scores")),
    Case(1, 2, 2, 129, 129, 384, F, F, 1, T, ("randn", "front_max")),
    # D > 128, transposed V: the transpose pre-pass in front of the natural-V kernel
    Case(2, 4, 2, 130, 776, 264, T, F, 1, F, ("randn", "tail_max")),
    Case(1, 2, 2, 130, 776, 136, T, T, 1, F, ("randn", "ramp_max", "future_max")),
    Case(1, 8, 2, 130, 776, 264, T, T, 1, F, ("randn", "one_hot", "diag_gather")),
    Case(2, 8, 2, 5, 776, 136, T, T, 1, F, ("randn", "neg_scores", "future_max")),
    Case(1, 8, 8, 1, 776, 136, T, F, 13, F, ("randn", "front_max")),
    Case(1, 8, 1, 130, 776, 264, T, T, 9, F, ("randn", "tail_max", "diag_gather")),
    Case(2, 4, 4, 5, 776, 136, T, T, 4, F, ("randn", "ramp_max", "future_max")),
    Case(1, 2, 2, 136, 136, 136, T, F, 1, T, ("randn", "one_hot")),
    Case(1, 2, 2, 136, 136, 512, T, F, 1, T, ("randn", "neg_scores")),
    # D = 520 / 776 / 1000: three slabs and four, a K/V ring shorter than one key block (776), the smallest ring
    # (1000): attn_ring_ref.  Last in the table, so that the rows above keep their places.
    Case(1, 8, 2, 130, 777, 776, F, T, 1, F, ("randn", "neg_scores", "future_max")),
    Case(2, 8, 2, 5, 1000, 1000, F, T, 1, F, ("randn", "front_max", "diag_gather")),
    Case(1, 8, 8, 130, 777, 1000, F, T, 5, F, ("randn", "ramp_max", "future_max")),
    Case(1, 4, 1, 1, 1000, 776, F, F, 17, F, ("randn", "tail_max")),
    Case(2, 4, 2, 130, 776, 1000, T, F, 1, F, ("randn", "one_hot")),
    Case(1, 8, 2, 130, 776, 520, T, T, 3, F, ("randn", "tail_max", "diag_gather")),
]

CASES = [(c, gen) for c in CASES_BY_SHAPE for gen in c.gens]


def case_key(c):
    return path(c.B, c.H, c.Hkv, c.Nq, c.Nk, c.D, c.vt, c.causal, c.splits, c.rms)[0]


def cases_by_key():
    """{path key: [(case, generator), ...]} of CASES."""
    out = {}
    for c, gen in CASES:
        out.setdefault(case_key(c), []).append((c, gen))
    return out
