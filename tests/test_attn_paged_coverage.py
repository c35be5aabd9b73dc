"""The paged dispatch restated in attn_paged_ref.py matches the built library, the GPU case table of
test_attn_paged_gpu.py reaches every path in every page-size regime, and every shape of tools/bench_attn_paged.py has a
GPU case at that shape."""
import importlib.util
import shutil
import subprocess
from pathlib import Path

import pytest
import torch

import attn_mask_ref as M
import attn_paged_ref as P

ROOT = Path(__file__).resolve().parent.parent


def _name(inst):
    return "attn_fwd_paged_kernel<%d, %d, %d, %s>" % (*inst[:3], ", ".join(str(x).lower() for x in inst[3:]))


INSTANTIATIONS = [
    "attn_fwd_paged_kernel<128, 64, 2, false, false>", "attn_fwd_paged_kernel<128, 64, 2, false, true>",
    "attn_fwd_paged_kernel<128, 64, 2, true, false>", "attn_fwd_paged_kernel<128, 64, 2, true, true>",
    "attn_fwd_paged_kernel<256, 64, 1, false, false>", "attn_fwd_paged_kernel<256, 64, 1, false, true>",
    "attn_fwd_paged_kernel<256, 64, 1, true, false>", "attn_fwd_paged_kernel<256, 64, 1, true, true>",
    "attn_fwd_paged_kernel<64, 128, 2, false, false>", "attn_fwd_paged_kernel<64, 128, 2, false, true>",
    "attn_fwd_paged_kernel<64, 128, 2, true, false>", "attn_fwd_paged_kernel<64, 128, 2, true, true>"]


def test_reachable_instantiations():
    assert len(P.reachable()) == 54
    assert {k[6] for k in P.reachable()} == {"<", "=", ">"}
    assert sorted(map(_name, {P.instantiation(k) for k in P.reachable()})) == INSTANTIATIONS


def test_library_has_exactly_the_reachable_instantiations(built_lib):
    from leetcuda_b200 import _capi
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not Path(cuobjdump).exists():
        pytest.skip("cuobjdump not available")
    sass = subprocess.run([cuobjdump, "-sass", str(_capi.LIB_PATH)], capture_output=True, text=True, check=True).stdout
    built = P.parse_instantiations(line for line in sass.splitlines() if "Function :" in line)
    assert len(built) == len(set(built)) == 12
    assert sorted(map(_name, built)) == INSTANTIATIONS


def _missing(cases):
    return P.reachable() - set(P.cases_by_key(cases))


def test_cases_reach_every_path():
    missing, extra = _missing(P.CASES), set(P.cases_by_key()) - P.reachable()
    assert not missing, "paths without a case in attn_paged_ref.CASES: " + "; ".join(map(str, sorted(missing)))
    assert not extra, "cases of paths reachable() does not list: " + "; ".join(map(str, sorted(extra)))


def test_removing_a_row_fails_the_gate():
    """The gate is sharp: the only row of a path taken out of the table leaves that path missing, by name."""
    by_key = P.cases_by_key()
    key = next(k for k, cs in by_key.items() if len({id(c) for c, _ in cs}) == 1)
    row = by_key[key][0][0]
    assert _missing([(c, g) for c, g in P.CASES if c is not row]) == {key}


def test_case_lengths_and_shapes():
    """Every row mixes the key lengths 0, 1, kBN +- 1, page_size +- 1 and the full padded length; the table covers
    G in {1, 4, 8}, every head dim of the kernel families and causal rows with Lq > Lk."""
    for c in P.CASES_BY_SHAPE:
        kbn, _ = M.kernel_shape(c.D)
        nk = c.page_size * c.max_pages
        assert {0, 1, kbn - 1, kbn + 1, c.page_size - 1, c.page_size + 1, nk} <= set(c.lk), c
        assert len(c.lq) == len(c.lk) and max(c.lq) == c.Nq and min(c.lq) <= 1, c
        assert nk <= 1000 and c.H <= 8, c
    assert {c.H // c.Hkv for c in P.CASES_BY_SHAPE} >= {1, 4, 8}
    assert {c.D for c in P.CASES_BY_SHAPE} >= {40, 64, 72, 128, 136, 264}
    assert any(c.causal and any(a > b for a, b in zip(c.lq, c.lk)) for c in P.CASES_BY_SHAPE)


@pytest.mark.parametrize("page_size", [16, 32, 64, 128, 256])
@pytest.mark.parametrize("kbn", [64, 128])
def test_sub_loads_read_the_mapped_rows(kbn, page_size):
    """The restated sub-loads of every key block land in 1024-byte steps, cover the block, read key t from row
    t % page_size of page table[t // page_size], and never read a table entry past the sequence's last page."""
    g = torch.Generator().manual_seed(kbn + page_size)
    for lk in (1, page_size - 1, page_size + 1, kbn + 1, 3 * kbn + 17, 1000):
        used = -(-lk // page_size)
        table = torch.randperm(4 * used, generator=g)[:used].tolist() + [-1] * 3
        for j in range(-(-lk // kbn)):
            loads = P.sub_loads(j, kbn, page_size, lk, table)
            r = min(page_size, kbn)
            assert [off for off, _, _ in loads] == [i * r * 128 for i in range(kbn // r)]
            assert all(off % 1024 == 0 for off, _, _ in loads)
            for off, row, pi in loads:
                assert pi < used
                for x in range(r):
                    t = j * kbn + off // 128 + x
                    if t < lk:
                        assert row + x == table[t // page_size] * page_size + t % page_size


def test_gather_restates_the_mapping():
    ps, Hkv, D = 16, 2, 8
    pool = torch.arange(5 * ps * Hkv * D, dtype=torch.float32).reshape(5, ps, Hkv, D)
    table = torch.tensor([[3, 0, -1], [4, 4, 2]], dtype=torch.int32)
    out = P.gather(pool, table, [20, 40], 48)
    for b, lk in enumerate((20, 40)):
        for t in range(48):
            want = pool[table[b, t // ps], t % ps] if t < lk else torch.zeros(Hkv, D)
            assert torch.equal(out[b, :, t], want), (b, t)


def _bench_shapes():
    spec = importlib.util.spec_from_file_location("bench_attn_paged", ROOT / "tools" / "bench_attn_paged.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.SHAPES, mod.PAGE_SIZES


def test_every_benchmarked_shape_has_a_gpu_case():
    import test_attn_paged_gpu as G
    shapes, pages = _bench_shapes()
    assert shapes and set(pages) == {16, 256}
    assert sorted(G.BENCH_SHAPES) == sorted(shapes), "a shape of tools/bench_attn_paged.py has no GPU case"
    assert set(G.BENCH_PAGE_SIZES) == set(pages)
