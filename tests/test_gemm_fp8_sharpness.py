"""The fp8 GEMM bound of gemm_fp8_ref.py is loose enough for the kernel's arithmetic under the stated tensor-core
assumption TC(P) and sharp enough to catch the mistakes a scaled GEMM tends to make.  CPU only, small shapes.

A restatement of the kernel's order (four TC(P) k32 steps into a fresh accumulator per k-block, fp32 promotion, the
recipe's scales, one rounding) must stay inside the bound on every generator, and be bit for bit OutT(C64) on the exact
ones.  Each mutation must break the bound, for every recipe and output type it applies to, on at least one generator.
"""
import math

import numpy as np
import pytest
import torch

import gemm_fp8_ref as R

M, N = 64, 136                      # N: one full 128-column tile and a ragged one
K_VALUES = (400, 2048)              # 400: three full k-blocks and a ragged one
CASES = [(r, od) for r in R.RECIPES for od in R.OUT_DTYPES]


def _ids(c):
    return f"{c[0]}-{str(c[1])[6:]}"


def _data(gen, recipe, K, seed):
    a, b, _ = R.make_inputs(gen, M, N, K, seed=seed)
    sa, sb = R.make_scales(recipe, M, N, K, pow2=gen in R.EXACT, seed=seed)
    return a, b, sa, sb


@pytest.mark.parametrize("case", CASES, ids=_ids)
def test_kernel_arithmetic_stays_inside_the_bound(case):
    recipe, od = case
    for K in K_VALUES:
        for i, gen in enumerate(R.GENERATORS):
            a, b, sa, sb = _data(gen, recipe, K, seed=10 * K + i)
            ref = R.reference(a, b, sa, sb, recipe)
            got = R.emulate(a, b, sa, sb, recipe, od)
            ratio = ((got - ref["c"]).abs() / R.bound(ref, od)).max().item()
            assert ratio <= 1.0, (gen, K, ratio)
            if gen in R.EXACT:
                assert torch.equal(got, R.rounded(ref, od).double()), (gen, K)


MUTATIONS = {
    "drop_block": R.RECIPES,
    "neighbour": ("row", "block"),          # tensor-wise scaling has one scale: no neighbour to mistake it for
    "no_epi_scale": R.RECIPES,
    "second_round": R.RECIPES,
}


@pytest.mark.parametrize("mutation,case", [(m, c) for m, rs in MUTATIONS.items() for c in CASES if c[0] in rs],
                         ids=lambda x: x if isinstance(x, str) else _ids(x))
def test_mutation_is_rejected(mutation, case):
    recipe, od = case
    K = 2048
    worst = {}
    for i, gen in enumerate(R.GENERATORS):
        a, b, sa, sb = _data(gen, recipe, K, seed=10 * K + i)
        ref = R.reference(a, b, sa, sb, recipe)
        got = R.emulate(a, b, sa, sb, recipe, od, mutation=mutation, j_drop=R.kblocks(K) - 1)
        worst[gen] = ((got - ref["c"]).abs() / R.bound(ref, od)).max().item()
    assert max(worst.values()) > 1.0, worst


@pytest.mark.parametrize("recipe", ["tensor", "row"])
@pytest.mark.parametrize("od", R.OUT_DTYPES, ids=lambda d: str(d)[6:])
def test_whole_k_accumulation_without_promotion_is_rejected(recipe, od):
    """One tensor-core accumulator over K = 16384 of `cancel` data: the running sum reaches ~K/2 |p| and every step's
    error is relative to it; with promotion each k-block starts from zero."""
    Mc, K = 16, 16384
    a, b, _ = R.make_inputs("cancel", Mc, N, K, seed=3)
    sa, sb = R.make_scales(recipe, Mc, N, K, pow2=False, seed=3)
    ref = R.reference(a, b, sa, sb, recipe)
    bd = R.bound(ref, od)
    ok = ((R.emulate(a, b, sa, sb, recipe, od) - ref["c"]).abs() / bd).max().item()
    bad = ((R.emulate(a, b, sa, sb, recipe, od, mutation="no_promotion") - ref["c"]).abs() / bd).max().item()
    assert ok <= 1.0 < bad, (ok, bad)


def test_code_table_matches_torch():
    codes = torch.arange(256, dtype=torch.uint8).view(R.E4)
    want = codes.double().numpy()
    got = R.E4M3_TABLE
    nan = np.isnan(want)
    assert (np.isnan(got) == nan).all() and nan.sum() == 2
    assert (got[~nan] == want[~nan]).all()
    assert got[0x7E] == 448 and got[0x01] == 2.0 ** -9


def test_exact_generators_stay_exact():
    """int data: every in-block partial below 2^10; promoted sums on the grid of the smallest scale below 2^24 up to
    K = 8192 for block scales (g in 2^-4 .. 2^4) and far beyond for tensor / row (the sum is an integer, scaled by
    powers of two after promotion).  The GPU tests use int data up to K = 4096."""
    a, b, _ = R.make_inputs("int", 8, 16, 4096)
    A, B = R.decode(a), R.decode(b)
    assert A.abs().max() <= 2 and B.abs().max() <= 2
    assert 128 * 4 < 2 ** 10
    assert 128 * 4 * R.kblocks(8192) * 2 ** 4 / 2 ** -4 < 2 ** 24
    sa, sb = R.make_scales("block", 8, 16, 4096, pow2=True)
    assert set(torch.log2(torch.cat([sa.flatten(), sb.flatten()])).tolist()) <= {-2, -1, 1, 2}


def test_tile_plan_restatement():
    p = R.tile_plan(1, 8, 16)
    assert (p["tiles_m"], p["tiles_n"], p["cs"], p["num_tiles"], p["kblocks"]) == (1, 1, 1, 1, 1)
    p = R.tile_plan(2600, 2344, 512)
    assert (p["tiles_m"], p["tiles_n"], p["cs"], p["num_tiles"]) == (21, 19, 2, 11 * 19)
    assert p["groups"] == [(0, 8), (8, 3)] and p["odd_tiles_m"]
    assert R.instantiation(torch.float16, "tensor") == R.instantiation(torch.float16, "row") == ("__half", False)
    assert R.instantiation(torch.bfloat16, "block") == ("__nv_bfloat16", True)


def test_kernel_constants_match_the_restatement():
    from pathlib import Path
    src = (Path(__file__).resolve().parent.parent / "leetcuda_b200" / "csrc" / "gemm_fp8_sm90.cuh").read_text()
    assert "constexpr int BN = 128;" in src and "constexpr int BK = 128;" in src
    assert "using C_ = hgemm::Cfg<BN>;" in src
    hg = (Path(__file__).resolve().parent.parent / "leetcuda_b200" / "csrc" / "hgemm_sm90.cuh").read_text()
    assert "STAGES = (kBN == 256) ? 4 : 6;" in hg and "constexpr int kGroupM = 16;" in hg
    assert R.STAGES == 6 and R.GROUP_M == 16 and math.isclose(R.U32, 2.0 ** -24)
