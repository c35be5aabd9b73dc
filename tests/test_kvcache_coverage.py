"""The KV-cache append's instantiations in the built library are exactly the restated set (kvcache_ref.INSTANTIATIONS),
their names stay clear of every other kernel family's patterns and name counters, the GPU case table reaches every
(T, cache type, layout, rotary) combination, and the benchmarked shapes have their GPU tests."""
import re
import shutil
import subprocess
from pathlib import Path

import pytest

import attn_bf16_ref as BF
import attn_fp8kv_ref as F8
import attn_paged_ref as P
import attn_paths as AP
import attn_seqlens_ref as S
import attn_varlen_ref as V
import kvcache_ref as K

ROOT = Path(__file__).resolve().parent.parent


def _sass_functions():
    from leetcuda_b200 import _capi
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not Path(exe).exists():
        pytest.skip("cuobjdump not available")
    out = subprocess.run([exe, "-sass", str(_capi.LIB_PATH)], capture_output=True, text=True, check=True).stdout
    return [line.split("Function :")[1].strip() for line in out.splitlines() if "Function :" in line]


def _demangled(names):
    r = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True)
    return r.stdout.splitlines() if r.returncode == 0 else []


def test_restated_instantiations():
    assert K.INSTANTIATIONS == [("bf16", "bf16"), ("bf16", "e4m3"), ("half", "e4m3"), ("half", "half")]
    assert K.name(("half", "e4m3")) == "kvcache_append_kernel<__half, __nv_fp8_e4m3>"


def test_library_has_exactly_the_restated_instantiations(built_lib):
    names = [n for n in _sass_functions() if "kvcache_append_kernel" in n]
    built = K.parse_instantiations(names)
    assert len(built) == len(set(built)) == len(names) == 4
    assert sorted(built) == K.INSTANTIATIONS
    dem = _demangled(names)
    if dem:
        assert sorted(K.parse_instantiations(dem)) == K.INSTANTIATIONS


def test_names_match_no_other_pattern_or_counter(built_lib):
    mangled = [n for n in _sass_functions() if "kvcache_append_kernel" in n]
    names = mangled + _demangled(mangled)
    for mod in (AP, S, P, BF, F8, V):
        assert not mod.parse_instantiations(names), mod.__name__
    for counter in ("attn_fwd_", "bf16_kernel", "fp8kv", "attn_combine_kernel", "attn_varlen_kernel"):
        assert not any(counter in n for n in names), counter


def test_cases_reach_every_combination():
    have = {K.combo(c) for c in K.CASES}
    assert have == K.combos() and len(K.combos()) == 32
    assert {c.D for c in K.CASES} == {64, 128, 256, 80}
    assert {c.n_new for c in K.CASES} == {1, 4, 130}
    assert {c.page_size for c in K.CASES if c.layout == "paged"} == {16, 256}
    assert {c.table_kind for c in K.CASES if c.layout == "paged"} == {"good", "bad"}
    assert {K.instantiation(c.T, c.cache) for c in K.CASES} == set(K.INSTANTIATIONS)
    for c in K.CASES:
        rd = K.rotary_dim(c)
        assert rd % 16 == 0 and 0 <= rd <= c.D and (c.rotary != "partial" or rd < c.D)
        assert c.cache != "e4m3" or c.D % 16 == 0
        # every row mixes an empty sequence, a clamped negative length, and a token dropped past capacity
        assert 0 in c.lens and min(c.lens) <= 0 and max(c.lens) + c.n_new > K.CAPACITY


def test_removing_a_case_fails_the_gate():
    rest = K.CASES[1:]
    assert {K.combo(c) for c in rest} != K.combos()


def test_bench_tool_shapes_agree():
    text = (ROOT / "tools" / "bench_kvcache.py").read_text()
    assert "K.BENCH_DECODE" in text and "K.BENCH_APPEND" in text and "K.bench_lengths" in text
    gpu = (ROOT / "tests" / "test_kvcache_gpu.py").read_text()
    assert re.search(r"def test_bench_decode_shape", gpu) and re.search(r"def test_bench_append_shape", gpu)
