"""The bf16 dispatch restated in attn_bf16_ref.py matches the built library, the GPU case table of test_attn_bf16_gpu.py
reaches every path of both bf16 kernels, and every shape of tools/bench_attn_bf16.py has a GPU case at that shape."""
import importlib.util
import shutil
import subprocess
from pathlib import Path

import pytest

import attn_bf16_ref as BF
import attn_paged_ref as P
import attn_seqlens_ref as S

ROOT = Path(__file__).resolve().parent.parent


def _name(inst):
    return "attn_fwd_%s_bf16_kernel<%d, %d, %d, %s>" % (*inst[:4], ", ".join(str(x).lower() for x in inst[4:]))


INSTANTIATIONS = [
    "attn_fwd_paged_bf16_kernel<128, 64, 2, false, false>", "attn_fwd_paged_bf16_kernel<128, 64, 2, false, true>",
    "attn_fwd_paged_bf16_kernel<128, 64, 2, true, false>", "attn_fwd_paged_bf16_kernel<128, 64, 2, true, true>",
    "attn_fwd_paged_bf16_kernel<256, 64, 1, false, false>", "attn_fwd_paged_bf16_kernel<256, 64, 1, false, true>",
    "attn_fwd_paged_bf16_kernel<256, 64, 1, true, false>", "attn_fwd_paged_bf16_kernel<256, 64, 1, true, true>",
    "attn_fwd_paged_bf16_kernel<64, 128, 2, false, false>", "attn_fwd_paged_bf16_kernel<64, 128, 2, false, true>",
    "attn_fwd_paged_bf16_kernel<64, 128, 2, true, false>", "attn_fwd_paged_bf16_kernel<64, 128, 2, true, true>",
    "attn_fwd_seqlens_bf16_kernel<128, 64, 2, false, false>", "attn_fwd_seqlens_bf16_kernel<128, 64, 2, false, true>",
    "attn_fwd_seqlens_bf16_kernel<128, 64, 2, true, false>", "attn_fwd_seqlens_bf16_kernel<128, 64, 2, true, true>",
    "attn_fwd_seqlens_bf16_kernel<256, 64, 1, false, false>", "attn_fwd_seqlens_bf16_kernel<256, 64, 1, false, true>",
    "attn_fwd_seqlens_bf16_kernel<256, 64, 1, true, false>", "attn_fwd_seqlens_bf16_kernel<256, 64, 1, true, true>",
    "attn_fwd_seqlens_bf16_kernel<64, 128, 2, false, false>", "attn_fwd_seqlens_bf16_kernel<64, 128, 2, false, true>",
    "attn_fwd_seqlens_bf16_kernel<64, 128, 2, true, false>", "attn_fwd_seqlens_bf16_kernel<64, 128, 2, true, true>"]


def test_reachable_instantiations():
    assert len(BF.reachable()) == len(S.reachable()) + len(P.reachable()) == 18 + 54
    assert sorted(map(_name, {BF.instantiation(k) for k in BF.reachable()})) == INSTANTIATIONS


def test_names_do_not_match_the_fp16_patterns():
    """The fp16 coverage tests pin their kernel sets by these patterns; no bf16 name may match them."""
    mangled = ["_ZN4b2004attn28attn_fwd_seqlens_bf16_kernelILi64ELi128ELi2ELb1ELb0EEEv",
               "_ZN4b2004attn26attn_fwd_paged_bf16_kernelILi64ELi128ELi2ELb1ELb0EEEv"]
    import attn_paths as AP
    for names in (INSTANTIATIONS, mangled):
        assert not S.parse_instantiations(names) and not P.parse_instantiations(names)
        assert not AP.parse_instantiations(names)
        assert not any("attn_fwd_kernel<" in n for n in names)
    assert len(BF.parse_instantiations(mangled)) == 2


def test_library_has_exactly_the_reachable_instantiations(built_lib):
    from leetcuda_b200 import _capi
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not Path(cuobjdump).exists():
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", str(_capi.LIB_PATH)], capture_output=True, text=True, check=True).stdout
    functions = [line for line in sass.splitlines() if "Function :" in line]
    built = BF.parse_instantiations(functions)
    assert len(built) == len(set(built)) == 24
    assert sorted(map(_name, built)) == INSTANTIATIONS
    assert sum("bf16_kernel" in f for f in functions) == 24
    assert sum("attn_combine_kernel" in f and "bfloat16" in f for f in functions) == 2


def test_cases_reach_every_path():
    keys = {BF.case_key(kind, c) for kind, c in BF.CASES if kind != "dense"}
    missing, extra = BF.reachable() - keys, keys - BF.reachable()
    assert not missing, "paths without a case in attn_bf16_ref.CASES: " + "; ".join(map(str, sorted(missing, key=str)))
    assert not extra, "cases of paths reachable() does not list: " + "; ".join(map(str, sorted(extra, key=str)))
    dense = {BF.case_key(kind, c, splits=c.splits or 2) for kind, c in BF.CASES if kind == "dense"}
    assert dense <= BF.reachable()
    assert {k[0] for k in dense} == {"seqlens"}, "a dense bf16 call runs the seqlens kernel"


def test_every_benchmarked_shape_has_a_gpu_case():
    spec = importlib.util.spec_from_file_location("bench_attn_bf16", ROOT / "tools" / "bench_attn_bf16.py")
    tool = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tool)
    import test_attn_bf16_gpu as G
    assert tool.SHAPES == G.BENCH_SHAPES
    assert tool.PAGE_SIZE == G.BENCH_PAGE_SIZE
    assert tool.LK_RANGE == (256, 8192)
    ids = [f"{G.BENCH_SHAPES[i][0].replace(' ', '-')}{i}" for i in range(len(G.BENCH_SHAPES))]
    assert len(set(ids)) == len(tool.SHAPES)
