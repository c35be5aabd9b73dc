"""The fp8-K/V dispatch restated in attn_fp8kv_ref.py matches the built library, the GPU case table of
test_attn_fp8kv_gpu.py reaches every path of both fp8 kernels for both Q/O types, and every shape of
tools/bench_attn_fp8kv.py has a GPU case at that shape."""
import importlib.util
import re
import shutil
import subprocess
from pathlib import Path

import pytest

import attn_bf16_ref as BF
import attn_fp8kv_ref as F
import attn_paged_ref as P
import attn_seqlens_ref as S

ROOT = Path(__file__).resolve().parent.parent
_CT = {"half": "__half", "bf16": "__nv_bfloat16"}


def _name(inst):
    kind, ds, bn, wg, causal, split, T = inst
    return f"attn_fwd_fp8kv_{kind}_kernel<{ds}, {bn}, {wg}, {str(causal).lower()}, {str(split).lower()}, {_CT[T]}>"


INSTANTIATIONS = sorted(
    f"attn_fwd_fp8kv_{kind}_kernel<{ds}, {bn}, {wg}, {c}, {s}, {t}>"
    for kind in ("paged", "seqlens") for ds, bn, wg in ((64, 128, 2), (128, 64, 2), (256, 64, 1))
    for c in ("false", "true") for s in ("false", "true") for t in ("__half", "__nv_bfloat16"))


def test_reachable_instantiations():
    assert len(F.reachable()) == 2 * len(BF.reachable()) == 144
    assert sorted(map(_name, {F.instantiation(k) for k in F.reachable()})) == INSTANTIATIONS
    assert len(INSTANTIATIONS) == 48


def _sass_functions():
    from leetcuda_b200 import _capi
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not Path(cuobjdump).exists():
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", str(_capi.LIB_PATH)], capture_output=True, text=True, check=True).stdout
    return [line for line in sass.splitlines() if "Function :" in line]


def test_library_has_exactly_the_reachable_instantiations(built_lib):
    functions = _sass_functions()
    built = F.parse_instantiations(functions)
    assert len(built) == len(set(built)) == 48
    assert sorted(map(_name, built)) == INSTANTIATIONS
    assert sum("fp8kv" in f for f in functions) == 48
    # the split combine stays in attn_capi.cu: two per output type
    assert sum("attn_combine_kernel" in f for f in functions) == 4


def test_names_do_not_match_the_existing_patterns(built_lib):
    """The fp16 and bf16 coverage tests pin their kernel sets by these patterns; no fp8 name may match them."""
    import attn_paths as AP
    names = [f for f in _sass_functions() if "fp8kv" in f] + INSTANTIATIONS
    assert len(names) == 96
    assert not S.parse_instantiations(names) and not P.parse_instantiations(names)
    assert not AP.parse_instantiations(names) and not BF.parse_instantiations(names)
    for pattern in ("attn_fwd_kernelILi", "attn_fwd_seqlens_kernelILi", "attn_fwd_paged_kernelILi",
                    r"attn_fwd_(seqlens|paged)_bf16_kernel", "bf16_kernel", "attn_fwd_kernel<"):
        assert not any(re.search(pattern, n) for n in names), pattern


def _missing(cases):
    keys = {F.case_key(T, kind, c) for T, kind, c in cases if c.splits != 0}
    return F.reachable() - keys, keys - F.reachable()


def test_cases_reach_every_path():
    missing, extra = _missing(F.CASES)
    assert not missing, "paths without a case in attn_fp8kv_ref.CASES: " + "; ".join(map(str, sorted(missing, key=str)))
    assert not extra, "cases of paths reachable() does not list: " + "; ".join(map(str, sorted(extra, key=str)))
    assert all(c.D % 16 == 0 for _, _, c in F.CASES)
    assert {F.case_key(T, k, c)[1] for T, k, c in F.CASES if k == "dense" and c.splits} == {"seqlens"}, \
        "a dense fp8 call runs the seqlens kernel"


def test_removing_a_paths_only_row_fails_by_name():
    """The gate names the path whose only row is gone."""
    rows = {}
    for i, (T, kind, c) in enumerate(F.CASES):
        if c.splits:
            rows.setdefault(F.case_key(T, kind, c), []).append(i)
    only = [(key, ix[0]) for key, ix in rows.items() if len(ix) == 1]
    assert only, "no path has a single row"
    for key, i in only[:8]:
        missing, _ = _missing(F.CASES[:i] + F.CASES[i + 1:])
        assert missing == {key}, (key, missing)


def _tool():
    spec = importlib.util.spec_from_file_location("bench_attn_fp8kv", ROOT / "tools" / "bench_attn_fp8kv.py")
    tool = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tool)
    return tool


def test_every_benchmarked_shape_has_a_gpu_case():
    tool = _tool()
    import test_attn_fp8kv_gpu as G
    assert tool.SHAPES == G.BENCH_SHAPES
    assert tool.LK_RANGE == G.BENCH_LK_RANGE == (256, 8192)
    for i in range(len(tool.SHAPES)):
        assert tool.lengths(i) == G.bench_lengths(i)
    ids = [G.BENCH_SHAPES[i][0].replace(" ", "-") for i in range(len(G.BENCH_SHAPES))]
    assert len(set(ids)) == len(tool.SHAPES)
    names = {s[0] for s in tool.SHAPES}
    assert {"dense decode", "seqlens decode", "paged decode p16", "paged decode p256", "long decode",
            "paged causal prefill"} == names
