"""The attention dispatch restated in attn_paths.py matches the built library, and the GPU case table runs every path
it can take.  A new template parameter or instantiation fails here until attn_paths.path and CASES cover it; a path
that drifts from the C++ dispatch fails the profiler check of test_attn_paths_gpu.py."""
import shutil
import subprocess
from pathlib import Path

import pytest

import attn_mask_ref as M
import attn_paths as P
import attn_ref as R


def _name(inst):
    return "attn_fwd_kernel<%d, %d, %d, %s>" % (*inst[:3], ", ".join(str(x).lower() for x in inst[3:]))


def test_reachable_instantiations():
    insts = {P.instantiation(k) for k in P.reachable()}
    assert len(P.reachable()) == 50
    assert sorted(map(_name, insts)) == [
        "attn_fwd_kernel<128, 64, 2, false, false, false, false>",
        "attn_fwd_kernel<128, 64, 2, false, false, false, true>",
        "attn_fwd_kernel<128, 64, 2, false, true, false, false>",
        "attn_fwd_kernel<128, 64, 2, false, true, true, false>",
        "attn_fwd_kernel<128, 64, 2, false, true, true, true>",
        "attn_fwd_kernel<128, 64, 2, true, false, false, false>",
        "attn_fwd_kernel<128, 64, 2, true, false, false, true>",
        "attn_fwd_kernel<128, 64, 2, true, true, false, false>",
        "attn_fwd_kernel<128, 64, 2, true, true, true, false>",
        "attn_fwd_kernel<128, 64, 2, true, true, true, true>",
        "attn_fwd_kernel<256, 64, 1, false, false, false, false>",
        "attn_fwd_kernel<256, 64, 1, false, false, false, true>",
        "attn_fwd_kernel<256, 64, 1, false, true, false, false>",
        "attn_fwd_kernel<256, 64, 1, false, true, true, false>",
        "attn_fwd_kernel<256, 64, 1, false, true, true, true>",
        "attn_fwd_kernel<64, 128, 2, false, false, false, false>",
        "attn_fwd_kernel<64, 128, 2, false, false, false, true>",
        "attn_fwd_kernel<64, 128, 2, false, true, false, false>",
        "attn_fwd_kernel<64, 128, 2, false, true, true, false>",
        "attn_fwd_kernel<64, 128, 2, false, true, true, true>",
        "attn_fwd_kernel<64, 128, 2, true, false, false, false>",
        "attn_fwd_kernel<64, 128, 2, true, false, false, true>",
        "attn_fwd_kernel<64, 128, 2, true, true, false, false>",
        "attn_fwd_kernel<64, 128, 2, true, true, true, false>",
        "attn_fwd_kernel<64, 128, 2, true, true, true, true>"]


def test_library_instantiations_are_the_reachable_ones(built_lib):
    from leetcuda_b200 import _capi
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not Path(cuobjdump).exists():
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", str(_capi.LIB_PATH)], capture_output=True, text=True, check=True).stdout
    built = set(P.parse_instantiations(line for line in sass.splitlines() if "Function :" in line))
    want = {P.instantiation(k) for k in P.reachable()}
    assert built == want, ("built but not reachable: " + ", ".join(sorted(map(_name, built - want)))
                           + "; reachable but not built: " + ", ".join(sorted(map(_name, want - built))))


def test_cases_reach_every_path():
    got = set(P.cases_by_key())
    missing, extra = P.reachable() - got, got - P.reachable()
    assert not missing, "paths without a case in attn_paths.CASES: " + "; ".join(map(str, sorted(missing)))
    assert not extra, "cases of paths reachable() does not list: " + "; ".join(map(str, sorted(extra)))


def test_cases_per_path():
    """Every path has a randn case and an adversarial one, a causal path also a diagonal probe; the shapes stay small."""
    adversarial = set(R.GENERATORS) - {"randn"}
    for key, cases in P.cases_by_key().items():
        gens = {g for _, g in cases}
        assert "randn" in gens and gens & adversarial, (key, gens)
        if key[4]:
            assert gens & set(M.PROBES), (key, gens)
    for c, _ in P.CASES:
        assert c.B <= 2 and c.H <= 8 and c.Nk <= 1000, c


def test_path_rules():
    """Spot checks of the restated dispatch against attn_capi.cu."""
    # split kernels are <.., causal, causal, true> for every G; a causal split with G = 1 tiles per head at Nq >= 128
    assert P.path(1, 8, 8, 130, 1000, 64, False, True, 4, False) == ((64, 128, 2, False, True, True, True, False,
                                                                       "-", "per-head"), 2)
    assert P.path(1, 8, 8, 1, 1000, 64, False, False, 4, False)[0][4:7] == (False, False, True)
    # unsplit causal MHA is the plain causal kernel, GQA the kGQA one
    assert P.path(1, 8, 8, 5, 64, 128, False, True, 1, False)[0][4:] == (True, False, False, False, "-", "-")
    assert P.path(1, 8, 2, 5, 64, 128, False, True, 1, False)[0][4:] == (True, True, False, False, "-", "packed")
    # the pre-pass turns vt off for the kernel and adds a launch
    assert P.path(1, 2, 2, 8, 8, 136, True, False, 1, False) == ((256, 64, 1, False, False, False, False, True,
                                                                   "-", "-"), 2)
    assert P.path(1, 2, 2, 8, 8, 520, True, True, 3, False)[1] == 3
    # the RMS norm: one slab a row, 384 / 512 a cluster; nowhere else
    assert P.path(1, 2, 2, 8, 8, 256, False, False, 1, True)[0][8] == "row"
    assert P.path(1, 2, 2, 8, 8, 384, True, False, 1, True)[0][7:9] == (True, "cluster")
    for args in [(1, 2, 2, 8, 8, 264, False, False, 1, True), (1, 2, 1, 8, 8, 64, False, False, 1, True),
                 (1, 2, 2, 8, 8, 64, False, True, 1, True), (1, 2, 2, 8, 16, 64, False, False, 1, True),
                 (1, 2, 2, 8, 8, 64, False, False, 2, True), (1, 2, 2, 8, 12, 64, True, False, 1, False)]:
        with pytest.raises(ValueError):
            P.path(*args)
