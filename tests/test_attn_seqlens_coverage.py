"""The per-sequence-length dispatch restated in attn_seqlens_ref.py matches the built library, and the GPU case table
of test_attn_seqlens_gpu.py reaches every path it can take."""
import shutil
import subprocess
from pathlib import Path

import pytest

import attn_mask_ref as M
import attn_ref as R
import attn_seqlens_ref as S


def _name(inst):
    return "attn_fwd_seqlens_kernel<%d, %d, %d, %s>" % (*inst[:3], ", ".join(str(x).lower() for x in inst[3:]))


INSTANTIATIONS = [
    "attn_fwd_seqlens_kernel<128, 64, 2, false, false>", "attn_fwd_seqlens_kernel<128, 64, 2, false, true>",
    "attn_fwd_seqlens_kernel<128, 64, 2, true, false>", "attn_fwd_seqlens_kernel<128, 64, 2, true, true>",
    "attn_fwd_seqlens_kernel<256, 64, 1, false, false>", "attn_fwd_seqlens_kernel<256, 64, 1, false, true>",
    "attn_fwd_seqlens_kernel<256, 64, 1, true, false>", "attn_fwd_seqlens_kernel<256, 64, 1, true, true>",
    "attn_fwd_seqlens_kernel<64, 128, 2, false, false>", "attn_fwd_seqlens_kernel<64, 128, 2, false, true>",
    "attn_fwd_seqlens_kernel<64, 128, 2, true, false>", "attn_fwd_seqlens_kernel<64, 128, 2, true, true>"]


def test_reachable_instantiations():
    assert len(S.reachable()) == 18
    assert sorted(map(_name, {S.instantiation(k) for k in S.reachable()})) == INSTANTIATIONS


def test_library_has_exactly_the_reachable_instantiations(built_lib):
    from leetcuda_b200 import _capi
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not Path(cuobjdump).exists():
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", str(_capi.LIB_PATH)], capture_output=True, text=True, check=True).stdout
    built = S.parse_instantiations(line for line in sass.splitlines() if "Function :" in line)
    assert len(built) == len(set(built)) == 12
    assert sorted(map(_name, built)) == INSTANTIATIONS


def _missing(cases):
    return S.reachable() - set(S.cases_by_key(cases))


def test_cases_reach_every_path():
    missing, extra = _missing(S.CASES), set(S.cases_by_key()) - S.reachable()
    assert not missing, "paths without a case in attn_seqlens_ref.CASES: " + "; ".join(map(str, sorted(missing)))
    assert not extra, "cases of paths reachable() does not list: " + "; ".join(map(str, sorted(extra)))


def test_removing_a_row_fails_the_gate():
    """The gate is sharp: the only row of a path taken out of the table leaves that path missing, by name."""
    by_key = S.cases_by_key()
    key = next(k for k, cs in by_key.items() if len({id(c) for c, _ in cs}) == 1)
    row = by_key[key][0][0]
    assert _missing([(c, g) for c, g in S.CASES if c is not row]) == {key}


def test_cases_per_path():
    """Every path has a randn case and an adversarial one, a causal path also a diagonal probe; every row mixes the
    key lengths 0, 1, kBN - 1, kBN, kBN + 1 and Nk and query lengths 0 or 1 with full ones."""
    adversarial = set(R.GENERATORS) - {"randn"}
    for key, cases in S.cases_by_key().items():
        gens = {g for _, g in cases}
        assert "randn" in gens and gens & adversarial, (key, gens)
        if key[3]:
            assert gens & set(M.PROBES), (key, gens)
    for c in S.CASES_BY_SHAPE:
        kbn, _ = M.kernel_shape(c.D)
        assert {0, 1, kbn - 1, kbn, kbn + 1, c.Nk} <= set(c.lk), c
        assert {0, 1, c.Nq} <= set(c.lq) or {1, c.Nq} <= set(c.lq), c
        assert len(c.lq) == len(c.lk) <= 8 and c.H <= 8 and c.Nk <= 1000, c
    assert any(c.causal and any(a > b for a, b in zip(c.lq, c.lk)) for c in S.CASES_BY_SHAPE)
    assert {c.H // c.Hkv for c in S.CASES_BY_SHAPE} >= {1, 4, 8}
    assert {c.D for c in S.CASES_BY_SHAPE} >= {40, 64, 72, 128, 136, 264}
