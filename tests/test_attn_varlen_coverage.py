"""The packed variable-length dispatch restated in attn_varlen_ref.py matches the built library, its kernels stay clear
of every other kernel family's patterns and counters, and the GPU case table of test_attn_varlen_gpu.py reaches every
instantiation."""
import shutil
import subprocess
from pathlib import Path

import pytest

import attn_bf16_ref as BF
import attn_fp8kv_ref as F8
import attn_mask_ref as M
import attn_paged_ref as P
import attn_paths as AP
import attn_ref as R
import attn_seqlens_ref as S
import attn_varlen_ref as V


def _cuobjdump():
    exe = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not Path(exe).exists():
        pytest.skip("cuobjdump not available")
    return exe


def _functions(flag):
    from leetcuda_b200 import _capi
    return subprocess.run([_cuobjdump(), flag, str(_capi.LIB_PATH)], capture_output=True, text=True,
                          check=True).stdout.splitlines()


def _demangled(names):
    r = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True)
    return r.stdout.splitlines() if r.returncode == 0 else []


def test_reachable_instantiations():
    assert len(V.reachable()) == 24
    assert len(V.INSTANTIATIONS) == 24
    assert "attn_varlen_kernel<64, 128, 2, false, false, __half>" in V.INSTANTIATIONS
    assert "attn_varlen_kernel<256, 64, 1, true, true, __nv_bfloat16>" in V.INSTANTIATIONS


def test_grid_restatement():
    assert V.tph(130, 64) == 2 and V.tph(128, 128) == 1 and V.tph(130, 264) == 3
    assert V.grid(8, 32, 8, 4096, 128) == (4 * 32, 64)
    assert V.grid(2, 8, 1, 130, 520) == (8 * 3 * 3, 2)
    assert V.grid(3, 4, 4, 1, 1024) == (1 * 1 * 4, 12)


def test_library_has_exactly_the_reachable_instantiations(built_lib):
    names = [line.split("Function :")[1].strip() for line in _functions("-sass") if "Function :" in line]
    built = V.parse_instantiations(names)
    assert len(built) == len(set(built)) == 24
    assert sorted(map(V.name, built)) == V.INSTANTIATIONS
    assert set(built) == V.reachable()


def test_names_match_no_other_pattern_or_counter(built_lib):
    """The varlen kernels are invisible to the other families' restated parsers and to the name counters of the
    existing coverage tests: attn_fwd_ (every attn_fwd_body kernel), bf16_kernel, fp8kv, attn_combine_kernel."""
    mangled = [line.split("Function :")[1].strip() for line in _functions("-sass")
               if "Function :" in line and "attn_varlen_kernel" in line]
    assert len(mangled) == 24
    names = mangled + _demangled(mangled)
    assert len(names) in (24, 48)
    for mod in (AP, S, P, BF, F8):
        assert not mod.parse_instantiations(names), mod.__name__
    for counter in ("attn_fwd_", "bf16_kernel", "fp8kv", "attn_combine_kernel"):
        assert not any(counter in n for n in names), counter


def test_no_static_shared_memory(built_lib):
    """Every varlen kernel takes only the dynamic shared memory sized like the seqlens kernels' (plus the 1 KiB the
    driver reserves per CTA on sm_90, which cuobjdump counts in SHARED)."""
    out = _functions("-res-usage")
    shared = {}
    for name, usage in zip(out, out[1:]):
        if name.strip().startswith("Function ") and "attn_varlen_kernel" in name:
            shared[name.split()[1].rstrip(":")] = int(usage.split("SHARED:")[1].split()[0])
    assert len(shared) == 24
    assert set(shared.values()) <= {0, 1024}, shared


def _missing(cases):
    return V.reachable() - set(V.cases_by_key(cases))


def test_cases_reach_every_instantiation():
    missing, extra = _missing(V.CASES), set(V.cases_by_key()) - V.reachable()
    assert not missing, "instantiations without a case in attn_varlen_ref.CASES: " + "; ".join(map(str, sorted(missing)))
    assert not extra, "cases of paths reachable() does not list: " + "; ".join(map(str, sorted(extra)))


def test_removing_a_row_fails_the_gate():
    """The gate is sharp: the only row of a path taken out of the table leaves that path missing, by name."""
    by_key = V.cases_by_key()
    key = next(k for k, cs in by_key.items() if len({id(c) for c, _ in cs}) == 1)
    row = by_key[key][0][0]
    assert _missing([(c, g) for c, g in V.CASES if c is not row]) == {key}


def test_cases_cover_the_edges():
    """Every path has a randn case and an adversarial one, a causal path also a diagonal probe; every row mixes
    Lq = 0, Lq > max_q, Lk = 0, Lk not a multiple of kBN and Lk > max_k; causal rows have Lq > Lk; the head dims cover
    every family and ring regime, G = 1 and G > 1."""
    adversarial = set(R.GENERATORS) - {"randn"}
    for key, cases in V.cases_by_key().items():
        gens = {g for _, g in cases}
        assert "randn" in gens and gens & adversarial, (key, gens)
        if key[3]:
            assert gens & set(M.PROBES), (key, gens)
    for c in V.CASES_BY_SHAPE:
        kbn, _ = M.kernel_shape(c.D)
        assert 0 in c.lq and max(c.lq) > c.max_q, c
        assert 0 in c.lk and {kbn - 1, kbn + 1} <= set(c.lk) and max(c.lk) > c.max_k, c
        if c.causal:
            assert any(a > b > 0 for a, b in zip(c.lq, c.lk)), c
    assert {c.D for c in V.CASES_BY_SHAPE} >= {8, 64, 72, 128, 136, 256, 520, 1024}
    assert {c.H // c.Hkv for c in V.CASES_BY_SHAPE} >= {1, 4, 8}
    assert {c.page_size for c in V.CASES_BY_SHAPE if c.paged} >= {16, 64, 128, 256}
