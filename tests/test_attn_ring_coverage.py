"""The K/V ring of the D > 128 attention kernels restated in attn_ring_ref.py, and the gate that keeps the GPU case
tables inside its hard regimes: for every kernel kind and element type, three slabs and four, a ring shorter than one
key block, the smallest ring, and the causal mask, splits, the zeroed partial key block and paged sub-loads in a ring
that wraps.  The path gates (test_attn_*_coverage.py) cannot see these: a path key records the kernel family, not the
head dim inside it."""
import shutil
import subprocess
from pathlib import Path

import pytest

import attn_fp8kv_ref as F
import attn_ring_ref as RR


def test_ring_restated():
    """The ring depths, slabs and chunks per key block of attn_ring_ref's docstring."""
    assert [RR.ring(D) for D in (136, 264, 520, 776, 1000, 1024)] == [16, 16, 16, 15, 12, 12]
    assert [RR.ring(D, fp8=True) for D in (144, 272, 528, 784, 1008, 1024)] == [16, 15, 12, 10, 8, 8]
    assert RR.smallest_ring(False) == 12 and RR.smallest_ring(True) == 8
    assert [RR.slabs(D) for D in (264, 520, 528, 776, 1000)] == [2, 3, 3, 4, 4]
    assert [RR.chunks_per_block(520, s) for s in range(3)] == [13, 13, 10]
    assert [RR.chunks_per_block(776, s) for s in range(4)] == [17, 17, 17, 14]
    assert [RR.chunks_per_block(1000, s) for s in range(4)] == [20, 20, 20, 20]
    assert [RR.chunks_per_block(528, s) for s in range(3)] == [13, 13, 10]
    # the first head dims whose ring holds less than one key block
    wraps = lambda D, fp8: RR.ring(D, fp8) < max(RR.chunks_per_block(D, s) for s in range(RR.slabs(D)))
    assert min(D for D in range(136, 1025, 8) if wraps(D, False)) == 776
    assert min(D for D in range(144, 1025, 16) if wraps(D, True)) == 528
    # every supported head dim fits: at least two slots, at most 227 KiB
    for D in range(136, 1025, 8):
        for fp8 in (False, True):
            if fp8 and D % 16:
                continue
            assert 2 <= RR.ring(D, fp8) <= 16 and RR.smem_bytes(D, fp8) <= 227 * 1024, (D, fp8)
    assert RR.smem_bytes(1000) == 16 * 8192 + 12 * 8192 + 8 * 25 + 256 + 1024
    assert RR.smem_bytes(1008, fp8=True) == 16 * 8192 + 8 * 8192 + 8 * 17 + 256 + 1024 + 8 * (64 * 64 + 8)


def test_attention_kernels_have_no_static_shared_memory(built_lib):
    """Every attention kernel takes only the dynamic shared memory fmha_dispatch sizes (and the 1 KiB the driver
    reserves per CTA on sm_90, which cuobjdump counts in SHARED), so a launch's shared memory is smem_bytes."""
    from leetcuda_b200 import _capi
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not Path(cuobjdump).exists():
        pytest.skip("cuobjdump not available")
    out = subprocess.run([cuobjdump, "-res-usage", str(_capi.LIB_PATH)], capture_output=True, text=True,
                         check=True).stdout.splitlines()
    shared = {}
    for name, usage in zip(out, out[1:]):
        if name.strip().startswith("Function ") and ("attn_fwd_" in name or "transpose_dn_to_nd" in name):
            shared[name.split()[1].rstrip(":")] = int(usage.split("SHARED:")[1].split()[0])
    attn = {k: v for k, v in shared.items() if "attn_fwd_" in k}
    assert len(attn) == 25 + 12 + 12 + 24 + 48
    reserve = {v for v in attn.values()}
    assert reserve <= {0, 1024}, reserve
    # the transpose pre-pass holds its 32 x 33 fp16 tile on top of the same reserve
    assert {v for k, v in shared.items() if "transpose_dn_to_nd" in k} == {2112 + min(reserve)}


def _message(missing):
    return "regimes without a row: " + "; ".join(f"{kind} {T}: {g}" for kind, T, g in sorted(missing))


def test_tables_reach_every_regime():
    rows = RR.table_rows()
    missing = RR.missing(rows)
    assert not missing, _message(missing)
    assert len(RR.KINDS) == 9


def test_removing_a_regimes_rows_fails_by_name():
    """For every regime of every kind: the table without the rows that reach it misses that regime."""
    rows = RR.table_rows()
    reached = {}
    for i, (kind, T, c) in enumerate(rows):
        for g in RR.regimes(kind, T, c):
            reached.setdefault((kind, T, g), []).append(i)
    assert set(reached) >= {(kind, T, g) for kind, T in RR.KINDS for g in RR.required(kind)}
    singles = 0
    for kind, T in RR.KINDS:
        for g in RR.required(kind):
            ix = set(reached[(kind, T, g)])
            singles += len(ix) == 1
            missing = RR.missing([r for i, r in enumerate(rows) if i not in ix])
            assert (kind, T, g) in missing and f"{kind} {T}: {g}" in _message(missing), (kind, T, g)
    assert singles, "no regime has a single row"


def test_regimes_of_a_row():
    """Spot checks of attn_ring_ref.regimes against the kernel's conditions."""
    import attn_paged_ref as P
    import attn_seqlens_ref as S
    c = S.Case(8, 2, 130, 777, 1000, True, 1, (130, 1), (0, 65), ())
    assert RR.regimes("seqlens", "half", c) == {RR.FOUR_SLABS, RR.WRAP, RR.SMALLEST, RR.WRAP_CAUSAL, RR.WRAP_PARTIAL}
    # no partial block below the padded Nk: a key length that is a multiple of kBN, or the padded Nk itself
    assert RR.WRAP_PARTIAL not in RR.regimes("seqlens", "half", c._replace(lk=(0, 64)))
    assert RR.WRAP_PARTIAL not in RR.regimes("seqlens", "half", c._replace(lk=(0, 777)))
    # ... or a sequence without a query
    assert RR.WRAP_PARTIAL not in RR.regimes("seqlens", "half", c._replace(lq=(130, 0)))
    # paged: every partial block is zeroed, the padded Nk included
    p = P.Case(8, 2, 5, 16, 50, 776, False, 3, (5, 5), (0, 790), ())
    assert RR.regimes("paged", "half", p) == {RR.FOUR_SLABS, RR.WRAP, RR.WRAP_SPLIT, RR.WRAP_PARTIAL, RR.WRAP_PAGE16}
    assert RR.regimes("paged", "bf16", p._replace(D=520, page_size=256, max_pages=3)) == {RR.THREE_SLABS}
    assert RR.regimes("paged", "fp8-bf16", p._replace(D=528, page_size=256, max_pages=3, lk=(0, 700))) == {
        RR.THREE_SLABS, RR.WRAP, RR.WRAP_SPLIT, RR.WRAP_PARTIAL, RR.WRAP_BIG_PAGE}
    assert RR.regimes("seqlens", "half", c._replace(D=264)) == set()


def test_fp8_cases_are_distinct():
    """fp8_dim maps no two rows of the fp16 / bf16 tables onto one fp8 row, and keeps their slab counts."""
    import attn_bf16_ref as BF
    assert len(F.CASES) == len(set(F.CASES))
    for kind, c in BF.CASES:
        assert RR.slabs(F.fp8_dim(c.D)) == RR.slabs(c.D) and RR.family(F.fp8_dim(c.D)) == RR.family(c.D), c
