"""The fp8 GEMM's instantiations in the built library are exactly the restated set (gemm_fp8_ref.INSTANTIATIONS), every
call maps onto one of them, and the GPU shape table reaches every launch regime: clusters of one and two, an odd
tiles_m, a partial raster group, several tiles per cluster, and the 6-stage ring wrapping across single-k-block tiles."""
import re
import shutil
import subprocess
from pathlib import Path

import pytest

import gemm_fp8_ref as R

ROOT = Path(__file__).resolve().parent.parent


def _sass_functions():
    from leetcuda_b200 import _capi
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not Path(exe).exists():
        pytest.skip("cuobjdump not available")
    out = subprocess.run([exe, "-sass", str(_capi.LIB_PATH)], capture_output=True, text=True, check=True).stdout
    return [line.split("Function :")[1].strip() for line in out.splitlines() if "Function :" in line]


def test_library_has_exactly_the_restated_instantiations(built_lib):
    names = [n for n in _sass_functions() if "gemm_e4m3_kernel" in n]
    built = R.parse_instantiations(names)
    assert len(built) == len(set(built)) == len(names) == 4
    assert sorted(built) == sorted(R.INSTANTIATIONS)
    assert not any("hgemm_wgmma_kernel" in n for n in names)


def test_every_call_has_an_instantiation():
    calls = {R.instantiation(od, r) for od in R.OUT_DTYPES for r in R.RECIPES}
    assert calls == set(R.INSTANTIATIONS)


def test_shapes_reach_every_launch_regime():
    plans = {s: R.tile_plan(*s) for s in R.SHAPES}
    for (M, N, K), p in plans.items():
        assert K % 16 == 0 and N % 8 == 0
    assert any(M == 1 for M, _, _ in R.SHAPES) and any(N == 8 for _, N, _ in R.SHAPES)
    assert any(K < R.BK for _, _, K in R.SHAPES)
    assert any(K % R.BK for _, _, K in R.SHAPES if K > R.BK)
    assert any(M % R.BM and N % R.BN for M, N, _ in R.SHAPES)
    assert {p["cs"] for p in plans.values()} == {1, 2}
    assert any(p["odd_tiles_m"] for p in plans.values())
    assert any(len(p["groups"]) > 1 and p["groups"][-1][1] < R.GROUP_M // 2 and p["groups"][-1][1] % 2
               for p in plans.values())                                     # a partial, odd raster group
    assert any(p["tiles_per_cluster"] >= 2 for p in plans.values())
    # single-k-block tiles, each cluster running more tiles than the ring has stages: the ring wraps across tiles
    assert any(p["kblocks"] == 1 and p["tiles_per_cluster"] > R.STAGES for p in plans.values())
    assert max(p["kblocks"] for p in plans.values()) >= 32


def test_bench_tool_and_gpu_tests_exist():
    tool = (ROOT / "tools" / "bench_gemm_fp8.py").read_text()
    for shape in ("8192, 8192, 8192", "2600, 2344, 4096", "4096, 28672, 8192", "4096, 8192, 28672"):
        assert shape in tool, shape
    gpu = (ROOT / "tests" / "test_gemm_fp8_gpu.py").read_text()
    for name in ("test_shape_matrix", "test_graph_replay_with_new_scales", "test_c_past_2_31_elements",
                 "test_8192_cubed_sampled_rows", "test_against_torch_scaled_mm", "test_kernel_name_under_profiler"):
        assert re.search(rf"def {name}\b", gpu), name
