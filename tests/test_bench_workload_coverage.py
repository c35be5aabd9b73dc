"""Every workload the benchmarks time has an entry in bench_workloads.WORKLOADS, every entry names a live workload, and
every entry points at tests that exist.  A new bench row, tool variant or shape fails here until it has an entry and a
check at its shape; a removed one fails until its entry goes."""
import ast

import bench_workloads as W


def _functions(rel):
    tree = ast.parse((W.ROOT / rel).read_text())
    return {n.name for n in tree.body if isinstance(n, ast.FunctionDef)}


def _gpu_case_kinds():
    """Keys of the `_HANDLERS` dict of the GPU module: the call kinds test_workload can run."""
    tree = ast.parse((W.ROOT / W.GPU_CASE.split("::")[0]).read_text())
    for node in tree.body:
        if isinstance(node, ast.Assign) and any(getattr(t, "id", None) == "_HANDLERS" for t in node.targets):
            return {k.value for k in node.value.keys}
    return set()


def test_every_workload_has_an_entry_and_every_entry_is_live():
    found = W.discovered()
    ids = [w.id for w in W.WORKLOADS]
    assert len(ids) == len(set(ids)), "duplicate ids: " + ", ".join(sorted({i for i in ids if ids.count(i) > 1}))
    missing = sorted(set(found) - set(ids))
    stale = sorted(set(ids) - set(found))
    assert not missing, "timed by the benchmarks but not in bench_workloads.WORKLOADS: " + ", ".join(missing)
    assert not stale, "in bench_workloads.WORKLOADS but no longer timed: " + ", ".join(stale)
    wrong = [f"{i}: the source calls {found[i]}, the table {W.BY_ID[i].call['op']}" for i in ids
             if found[i] is not None and found[i] != W.BY_ID[i].call["op"]]
    assert not wrong, "; ".join(wrong)


def test_pinned_shapes_and_calls_are_still_in_the_sources():
    for rel, literals in W.PINNED.items():
        text = W.source(rel)
        gone = [s for s in literals if s not in text]
        assert not gone, f"{rel} no longer contains: " + " | ".join(gone)


def test_every_check_resolves_to_a_test_function():
    kinds = _gpu_case_kinds()
    assert kinds, "test_bench_workloads_gpu.py has no _HANDLERS"
    for w in W.WORKLOADS:
        assert w.check, f"{w.id}: no check"
        for node in w.check:
            rel, name = node.split("::")
            assert (W.ROOT / rel).exists(), f"{w.id}: {rel} does not exist"
            assert name in _functions(rel), f"{w.id}: {node} is not a test function"
            if node == W.GPU_CASE:
                assert w.call["kind"] in kinds, f"{w.id}: test_workload has no case of kind {w.call['kind']!r}"
        if w.call["kind"] == "existing":
            assert W.GPU_CASE not in w.check, w.id
        else:
            assert W.GPU_CASE in w.check, f"{w.id}: kind {w.call['kind']!r} is checked in the GPU module"


def test_seqlens_lengths_are_the_tools_draw():
    """Lengths inside the tool's ranges, Lq = Lk for prefill, Lq = Nq for decoding, and the draw's first values."""
    lens = W.seqlens_lengths()
    assert len(lens) == len(W.SEQLENS.SHAPES)
    for (name, B, H, Hkv, Nq, Nk, D, causal, (lo, hi)), (lq, lk) in zip(W.SEQLENS.SHAPES, lens):
        assert len(lq) == len(lk) == B and all(lo <= x <= hi <= Nk for x in lk)
        assert lq == (lk if name == "causal prefill" else (Nq,) * B)
    import numpy as np
    rng = np.random.default_rng(0)
    name, B, *_, (lo, hi) = W.SEQLENS.SHAPES[0]
    assert lens[0][1] == tuple(int(x) for x in rng.integers(lo, hi + 1, size=B))


def test_auto_splits_restatement_spot_checks():
    """The restated rule on 132 SMs gives the split counts the README reports for the tools' shapes."""
    got = [W.auto_splits(B, H, Hkv, Nq, Nk, D, 132) for _, B, H, Hkv, Nq, Nk, D, _ in W.DECODE.SHAPES]
    assert got == [16, 2, 1, 1, 2, 1, 1]
    name, B, H, Hkv, Nq, Nk, D, *_ = W.SEQLENS.SHAPES[1]
    assert W.auto_splits(B, H, Hkv, Nq, Nk, D, 132) == 4
    assert W.auto_splits(1, 8, 8, 1, 64 * 15, 128, 132) == 1          # 15 key blocks: below the split threshold
    assert W.auto_splits(1, 8, 8, 1, 64 * 16, 128, 132) == 4          # 16 blocks, 4 per split
    assert W.auto_splits(1, 1, 1, 1, 64 * 4096, 128, 132) == 64       # capped at 64
