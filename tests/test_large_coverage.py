"""CPU gate over the large-tensor case table (large_ref.py): every family and entry point has a case, every case marked
past 2^31 checks a region whose restated element offset is >= 2^31 and byte offset >= 2^32 (so an int32 element or
byte offset would wrap inside the checked rows), and every case fits in 20 GiB.  Each check returns the names it
misses, so taking a family's only case out fails with that family's name."""
from __future__ import annotations

import pytest

import large_ref as L


def missing_families(cases):
    have = {c.family for c in cases}
    return sorted(f for f in L.FAMILIES if f not in have)


def missing_entries(cases):
    have = {(c.family, c.entry) for c in cases}
    return sorted(f"{f}:{e}" for f, es in L.ENTRIES.items() for e in es if (f, e) not in have)


def not_past(cases):
    """Cases marked past 2^31 whose offsets do not show it in one buffer."""
    bad = []
    for c in cases:
        if c.past and not any(off >= L.TWO31 and off * size >= L.TWO32 for _, off, size in c.offsets):
            bad.append(c.name)
    return bad


def families_not_past(cases):
    """Families (other than the grid edge) without a case past 2^31."""
    have = {c.family for c in cases if c.past}
    return sorted(f for f in L.FAMILIES if f != "grid_edge" and f not in have)


def over_limit(cases):
    return [f"{c.name}: {c.total / L.GiB:.2f} GiB" for c in cases if c.total > L.PEAK_LIMIT]


def test_every_family_has_a_case():
    assert not missing_families(L.CASES)


def test_every_entry_has_a_case():
    assert not missing_entries(L.CASES)


def test_past_cases_pass_2_31_elements_and_2_32_bytes():
    assert not not_past(L.CASES)
    assert not families_not_past(L.CASES)


def test_peaks_fit():
    assert not over_limit(L.CASES)


def test_names_unique_and_families_known():
    assert len(L.by_name()) == len(L.CASES)
    assert {c.family for c in L.CASES} <= set(L.FAMILIES)
    for c in L.CASES:
        assert c.entry in L.ENTRIES[c.family], c.name


@pytest.mark.parametrize("family", sorted(L.FAMILIES))
def test_gate_names_a_removed_family(family):
    """Without its cases the gate fails and names the family."""
    rest = [c for c in L.CASES if c.family != family]
    assert missing_families(rest) == [family]
    assert any(m.startswith(family + ":") for m in missing_entries(rest))


def test_gate_catches_a_case_below_2_31():
    """A past case whose region stays below 2^31 elements (here: the first batch of the dense case) is named."""
    c = L.by_name()["dense_f16_gqa_causal"]
    s = c.shape
    first = s["H"] * s["Nq"] * s["D"] - 1
    shrunk = L.Case(c.name, c.family, c.entry, c.dtype, s, c.peak, (("q", first, 2),), True)
    assert not_past([shrunk]) == [c.name]


def test_dense_layout_restated():
    """The dense case's largest Q offset from the layout (b*H + h)*N*D + t*D + d at b, h, t, d all last, and the batch
    that straddles 2^31."""
    c = L.by_name()["dense_f16_gqa_causal"]
    B, H, N, D = (c.shape[k] for k in ("B", "H", "Nq", "D"))
    off = ((B - 1) * H + H - 1) * N * D + (N - 1) * D + D - 1
    assert dict((n, o) for n, o, _ in c.offsets)["q"] == off
    b = L.TWO31 // (H * N * D)
    assert b * H * N * D < L.TWO31 <= (b + 1) * H * N * D < B * H * N * D


def test_paged_layout_restated():
    """(page * page_size + r) * Hkv * D + h * D + d at the pool's last page, row, head and column."""
    for name in ("paged_f16", "paged_bf16", "fp8_paged_f16"):
        c = L.by_name()[name]
        s = c.shape
        off = ((s["num_pages"] - 1) * s["page_size"] + s["page_size"] - 1) * s["Hkv"] * s["D"] + \
            (s["Hkv"] - 1) * s["D"] + s["D"] - 1
        assert dict((n, o) for n, o, _ in c.offsets)["k_pool"] == off
        # the top page pages the tables use lie past 2^31 elements (fp8: past 2^32 bytes)
        size = L.ELEM[s["kv"]]
        assert (s["num_pages"] - 1) * s["page_size"] * s["Hkv"] * s["D"] * size >= (L.TWO32 if size == 1 else L.TWO31)


def test_split_workspace_passes_4_gib():
    """The split row's fp32 workspace [S, B*H*Nq, D] passes 2^32 bytes: the combine kernel's 32-bit pack index runs
    over a buffer addressed past 4 GiB."""
    c = L.by_name()["dense_f16_split2"]
    s = c.shape
    q = s["B"] * s["H"] * s["Nq"] * s["D"]
    assert q == 2 ** 29 + 2 ** 20
    ws = dict((n, (o, e)) for n, o, e in c.offsets)["ws_o"]
    assert (ws[0] + 1) * ws[1] > L.TWO32
    assert q // 8 + 256 < 0xFFFFFFFF                 # launch_combine's 32-bit pack index: 8 elements per pack


def test_long_context_head_passes_2_31():
    """The keys the GPU case makes dominant (rows tail .. Nk - 1) are exactly the ones at element offsets >= 2^31."""
    c = L.by_name()["long_context_f16"]
    s = c.shape
    assert s["Nk"] == 2 ** 24 + 77 and s["Hkv"] == 1
    assert (s["tail"] - 1) * s["D"] < L.TWO31 <= s["tail"] * s["D"] and s["tail"] < s["Nk"]
    assert set(s["splits"]) == {1, 64}


def test_fp8_and_varlen_paged_rows():
    """fp8 K/V past 2^32 bytes both paged and as a padded cache; varlen over a paged pool past 2^31 elements."""
    by = L.by_name()
    for name in ("fp8_paged_f16", "fp8_seqlens_f16"):
        c = by[name]
        assert c.shape["kv"] == "e4m3" and c.past and (c.shape["k_scale"], c.shape["v_scale"]) != (1.0, 1.0)
    c = by["varlen_paged_f16"]
    s = c.shape
    assert s["num_pages"] * s["page_size"] * s["Hkv"] * s["D"] > L.TWO31 and c.past
    assert s["lk"][-1] == s["max_pages"] * s["page_size"]          # the last sequence reads the pool's last page


def test_sgemm_k_edges():
    """K = 2,097,216 lies past the transpose's old grid limit of 65535 k-tiles, K = 2,097,120 exactly on it."""
    ks = {c.shape["K"] for c in L.CASES if c.family == "sgemm"}
    assert L.TRANSPOSE_K_LIMIT == 2_097_120
    assert 2_097_216 in ks and 2_097_120 in ks
    longk = [c for c in L.CASES if c.shape.get("K") == 2_097_216]
    assert {c.shape["mode"] for c in longk} == {"tf32", "3xtf32"}
    assert {c.shape["round"] for c in longk if c.shape["mode"] == "tf32"} == {True, False}
    assert any(c.shape["gen"] == "tail" for c in longk)
    # {-1, 0, 1} inputs: every partial sum stays below 2^24, so C is the exact integer product
    assert max(c.shape["K"] for c in longk) < 2 ** 24


def test_grid_edge_at_65535():
    for c in L.CASES:
        if c.family == "grid_edge":
            assert c.shape["B"] * c.shape["Hkv"] == 65535, c.name
    assert {c.shape["kind"] for c in L.CASES if c.family == "grid_edge"} == {"dense", "seqlens", "paged", "varlen"}


def test_hgemm_rows_offset():
    c = L.by_name()["hgemm_f16_rows"]
    assert c.shape["row0"] * c.shape["N"] > L.TWO31
