"""The GEMM error bounds of gemm_ref.py are sharp enough to catch the mistakes a kernel rewrite tends to make, and loose
enough for the kernel's own arithmetic.  CPU only (numpy and the C oracle), at small shapes.

For each mode, every mutation below applied to the fp64 reference computation must break that mode's bound on at least
one of the generators the GPU tests use; restatements of the kernel's arithmetic (k16 steps with an fp32 accumulator,
oracle.hgemm_f16acc, oracle.sgemm_tf32, the hi/lo 3xTF32 split) must stay inside it on all of them.
"""
import re
from pathlib import Path

import numpy as np
import pytest

import gemm_ref as R
from oracle import oracle as O

M, N = 64, 264                                            # N: two full 128-column tiles and a ragged one
K_VALUES = {"f16": (72, 512, 2048), "tf32": (36, 512, 2048)}   # 72 / 36: one full k-block and a partial one
BN = 128


def _ks(mode):
    return K_VALUES["f16" if R.is_fp16(mode) else "tf32"]


def _cases(mode):
    dtype = np.float16 if R.is_fp16(mode) else np.float32
    for K in _ks(mode):
        for i, gen in enumerate(R.GENERATORS):
            a, b, _ = R.make_inputs(gen, M, N, K, dtype, seed=10 * K + i)
            yield gen, K, a, b


# ------------------------------------------------------------------ restatements of the kernel's arithmetic
def _f16_k16_fp32_acc(a, b):
    """One exact k16 step at a time into an fp32 accumulator (one rounding per add), C rounded once to fp16."""
    acc = np.zeros((a.shape[0], b.shape[1]), np.float32)
    for k in range(0, a.shape[1], 16):
        acc = acc + (a[:, k:k + 16].astype(np.float64) @ b[k:k + 16].astype(np.float64)).astype(np.float32)
    return acc.astype(np.float16)


def _split(x):
    hi = R.tf32(x)
    return hi, R.tf32(x - hi)


def _3xtf32(a, b, with_lo_hi=True):
    """The split of b200_sgemm_3xtf32: A' = [hi | hi | lo], B' = [hi ; lo ; hi], one TF32 GEMM over 3K."""
    ha, la = _split(a)
    hb, lb = _split(b)
    if not with_lo_hi:
        la = np.zeros_like(la)
    return O.sgemm_tf32(np.hstack([ha, ha, la]), np.vstack([hb, lb, hb]), mode="asis")


RESTATEMENTS = {
    "f16": _f16_k16_fp32_acc,
    "f16acc": lambda a, b: O.hgemm_f16acc(a, b, k_chunk=16),
    "tf32": lambda a, b: O.sgemm_tf32(a, b, mode="rna"),
    "tf32t": lambda a, b: O.sgemm_tf32(a, b, mode="trunc"),
    "3xtf32": _3xtf32,
}


# ------------------------------------------------------------------ mutations
def _product(a, b, mode):
    a64, b64 = R.operands(a, b, mode)
    return a64 @ b64


def _drop_last_kblock(a, b, mode):
    K = a.shape[1]
    kb = R.KBLOCK[mode]
    if K % kb == 0:
        return None
    keep = K - K % kb
    return _product(a[:, :keep], b[:keep], mode)


def _leak_past_k(a, b, mode):
    # the zero-filled k past K reads the next row of memory instead: here k = 0 once more
    return _product(np.hstack([a, a[:, :1]]), np.vstack([b, b[:1]]), mode)


def _swap_k_in_a(a, b, mode):
    a = a.copy()
    a[:, [1, 2]] = a[:, [2, 1]]                 # inside one 16-byte swizzle chunk (8 fp16, 4 fp32)
    return _product(a, b, mode)


def _swap_rows(a, b, mode):
    c = _product(a, b, mode)
    c[[3, 11]] = c[[11, 3]]
    return c


def _swap_cols(a, b, mode):
    c = _product(a, b, mode)
    c[:, [2, 10]] = c[:, [10, 2]]
    return c


def _tile_from_neighbour(a, b, mode):
    c = _product(a, b, mode)
    c[:, :BN] = c[:, BN:2 * BN]
    return c


def _f16acc_as_f16(a, b, mode):
    return O.hgemm_f16acc(a, b, k_chunk=16).astype(np.float64)


def _rounding_skipped(a, b, mode):
    return _product(a, b, "tf32t")


def _3xtf32_without_lo_hi(a, b, mode):
    return _3xtf32(a, b, with_lo_hi=False).astype(np.float64)


ALL = R.MODES
MUTATIONS = {
    "last_partial_kblock_dropped": (ALL, _drop_last_kblock),
    "k_leaked_past_K": (ALL, _leak_past_k),
    "k_pair_swapped_in_A": (ALL, _swap_k_in_a),
    "rows_r_r8_swapped": (ALL, _swap_rows),
    "cols_c_c8_swapped": (ALL, _swap_cols),
    "tile_holds_n_neighbour": (ALL, _tile_from_neighbour),
    "f16_accumulation": (("f16",), _f16acc_as_f16),
    "tf32_rounding_skipped": (("tf32",), _rounding_skipped),
    "3xtf32_without_lo_a_hi_b": (("3xtf32",), _3xtf32_without_lo_hi),
}


@pytest.mark.parametrize("mode", R.MODES)
def test_kernel_arithmetic_stays_inside_the_bound(mode):
    worst = {}
    for gen, K, a, b in _cases(mode):
        ref = R.reference(a, b, mode)
        bound = R.bound(ref)
        got = RESTATEMENTS[mode](a, b).astype(np.float64)
        err = np.abs(got - ref["c"])
        assert np.all(err <= bound), (gen, K, (err / bound).max())
        if gen in R.EXACT:
            assert np.array_equal(got, ref["c"]), (gen, K)
        worst[(gen, K)] = (err / bound).max()
    print(f"\n{mode}: largest |err|/bound of the restatement: "
          + ", ".join(f"{g}@K={k} {r:.3f}" for (g, k), r in worst.items()))
    assert max(worst.values()) > 0.02, "the bound is far looser than the arithmetic it covers"


@pytest.mark.parametrize("mode,mutation", [(m, n) for n, (modes, _) in MUTATIONS.items() for m in modes])
def test_mutation_is_rejected(mode, mutation):
    _, mutate = MUTATIONS[mutation]
    caught, worst = [], 0.0
    for gen, K, a, b in _cases(mode):
        ref = R.reference(a, b, mode)
        got = mutate(a, b, mode)
        if got is None:
            continue
        r = (np.abs(got - ref["c"]) / R.bound(ref)).max()
        worst = max(worst, r)
        if r > 1:
            caught.append(f"{gen}@K={K}")
    assert caught, f"no generator catches {mutation} in mode {mode}"
    print(f"{mode}: {mutation} rejected by {', '.join(caught)} (largest |err|/bound {worst:.3g})")


def test_tile_choice_restatement():
    """tile_width restates hgemm_impl; the shapes the docstrings of the GPU tests rely on, on 132 SMs."""
    t = R.tile_width(2600, 2000, 132)
    assert (t["bn"], t["tiles"], t["tiles_per_cta"]) == (128, 336, 3)
    assert t["groups"][-1] == (16, 5, True)
    t = R.tile_width(2600, 2344, 132)
    assert (t["bn"], t["tiles"], t["tiles_per_cta"]) == (256, 210, 2)
    assert R.tile_width(4096, 4096, 132)["bn"] == 256 and R.tile_width(256, 4096, 132)["bn"] == 128
    assert R.tile_width(3000, 120, 132)["bn"] == 256         # equal tile counts: the 0.9 factor keeps 256
    assert R.tile_width(8192, 8192, 132)["tiles_per_cta"] == 16
    # one k-block per tile on more tiles per CTA than the ring has slots, at both widths
    t = R.tile_width(8192, 4096, 132)
    assert (t["bn"], t["tiles_per_cta"]) == (256, 8) and 8 > R.STAGES[256]
    t = R.tile_width(8576, 1416, 132)
    assert (t["bn"], t["tiles_per_cta"]) == (128, 7) and 7 > R.STAGES[128]


def test_ring_depth_matches_the_kernel():
    src = (Path(__file__).resolve().parents[1] / "leetcuda_b200" / "csrc" / "hgemm_sm90.cuh").read_text()
    deep, shallow = re.search(r"STAGES = \(kBN == 256\) \? (\d+) : (\d+);", src).groups()
    assert R.STAGES == {256: int(deep), 128: int(shallow)}


def test_tf32_helper_matches_the_oracle():
    x = np.random.default_rng(3).standard_normal(4096).astype(np.float32) * np.float32(1e3)
    special = np.array([0x00000000, 0x80000000, 0x00000001, 0x007FFFFF, 0x00001000, 0x7F7FFFFF, 0xFF7FFFFF,
                        0x7F800000, 0xFF800000, 0x7FC00000, 0x7FC01234, 0x7F800001, 0xFFFFFFFF, 0x3F801000,
                        0xBF801000, 0x3F800FFF], np.uint32)
    x = np.concatenate([x, special.view(np.float32)])
    for trunc in (False, True):
        assert np.array_equal(R.tf32(x, trunc).view(np.uint32), O.tf32_round(x, trunc).view(np.uint32))


def test_tf32_oracle_on_nan_and_overflow_follows_the_instruction():
    """cvt.rna.tf32.f32 as recorded on an H100 (sm_90): NaN payloads are truncated, not rounded, so a NaN whose payload
    lies only in the 13 dropped bits becomes inf; the largest finite float rounds up to inf."""
    seen = {0x7FC01234: 0x7FC00000, 0x7F800001: 0x7F800000, 0x7FFFFFFF: 0x7FFFE000, 0xFFC00000: 0xFFC00000,
            0x7F7FFFFF: 0x7F800000, 0x7F7FEFFF: 0x7F7FE000, 0x00001000: 0x00002000, 0x00000FFF: 0x00000000}
    x = np.array(list(seen), np.uint32).view(np.float32)
    assert O.tf32_round(x).view(np.uint32).tolist() == list(seen.values())
