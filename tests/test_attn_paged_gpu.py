"""Paged K/V (b200_fmha_fwd_f16_paged, flash_attn.fmha_fwd(block_table=)) on the GPU, over every path and page-size
regime of attn_paged_ref.CASES_BY_SHAPE.

Every case scatters its padded K / V into a pool through a random page permutation and poisons what no sequence may
read: unused pool pages and the rows past Lk_b hold NaN, +Inf, -Inf or 65504 (in turn over the rows and generators),
table entries past each sequence's pages are -1, INT_MIN or ids of poisoned pages (in turn over the sequences), Q rows
>= Lq_b hold NaN, and O / lse sit inside NaN guard bands.  Checked:
  * bit for bit fmha_fwd(seqlens_q=, seqlens_k=) on the padded buffers, split or not (both pick the same split count:
    it follows the same padded shape);
  * the fp64 reference with each sequence's visibility (attn_seqlens_ref.reference / part_references,
    attn_split_ref.combine_bound when split); padded rows and rows without a key exactly O = 0, lse = -inf; the pool
    and the table come back unchanged;
  * _capi.launch_count() up by 1 unsplit, 2 split; under torch.profiler (in a child process) the restated
    attn_fwd_paged_kernel<...>, the combine exactly when it splits.
Then pages shared between sequences, a 65536-key sequence in 16-key pages among short ones, CUDA graphs replayed with
new tables and lengths, a side stream, every shape of tools/bench_attn_paged.py at full size, and SDPA with an
explicit mask.  The largest |err| / bound per path is printed at the end of the module (pytest -s).
"""
import collections
import math
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import attn_mask_ref as M
import attn_paged_ref as P
import attn_ref as R
import attn_seqlens_ref as S
import attn_split_ref as SR
from leetcuda_b200 import _capi, flash_attn
from test_attn_gqa_gpu import _inputs
from test_attn_numerics_gpu import _assert_margins, _guarded
from test_attn_seqlens_gpu import _kernels_per_call, _lens, _poison, profiled_names_of

pytestmark = pytest.mark.gpu

# the shapes and page sizes of tools/bench_attn_paged.py (test_attn_paged_coverage checks that they agree)
BENCH_SHAPES = [
    ("decode", 32, 32, 8, 1, 8192, 128, False, (256, 8192)),
    ("decode", 4, 64, 8, 1, 32768, 128, False, (1024, 32768)),
    ("causal prefill", 8, 32, 8, 4096, 4096, 128, True, (512, 4096)),
]
BENCH_PAGE_SIZES = (16, 256)

_ratios = collections.defaultdict(float)
_POISON = (float("nan"), float("inf"), float("-inf"), 65504.0)
_INT_MIN = -2 ** 31


def label(key):
    ds, bn, wg, causal, split, tiling, regime = key
    flags = [f for f, on in (("causal", causal), ("split", split)) if on]
    return f"<{','.join([str(ds), str(bn), str(wg)] + flags)}> {tiling} page{regime}kBN"


@pytest.fixture(scope="module", autouse=True)
def _report():
    t0 = time.time()
    yield
    if _ratios:
        print("\nlargest |err| / bound per path (attn_ref.o_bound / lse_bound, attn_split_ref.combine_bound):")
        for key in sorted({k for k, _ in _ratios}, key=str):
            print(f"  {label(key):<40} O {_ratios[(key, 'O')]:.3f}  lse {_ratios[(key, 'lse')]:.3f}")
    print(f"module time {time.time() - t0:.1f} s")


def paginate(k, v, lk, page_size, max_pages, poison, seed, pad=None):
    """Pools [num_pages, page_size, Hkv, D] holding the padded k, v [B,Hkv,Nk,D] in randomly placed pages (the last used
    page of a sequence keeps the padded rows past Lk_b), every unused page filled with `poison`, and the table
    [B, max_pages].  Entries past a sequence's pages: `pad`, or in turn over the sequences -1, INT_MIN and ids of
    unused pages."""
    B, Hkv, _, D = k.shape
    used = [-(-x // page_size) for x in lk]
    n_used = sum(used)
    num_pages = n_used + max(4, n_used // 4)
    perm = torch.randperm(num_pages, generator=torch.Generator().manual_seed(seed))
    pools = [torch.full((num_pages, page_size, Hkv, D), poison, dtype=torch.float16, device="cuda") for _ in range(2)]
    free = perm[n_used:]
    table = torch.empty(B, max_pages, dtype=torch.int32)
    n = 0
    for b in range(B):
        ids = perm[n:n + used[b]]
        n += used[b]
        rest = max_pages - used[b]
        table[b, :used[b]] = ids.int()
        fill = pad if pad is not None else (-1, _INT_MIN, None)[b % 3]
        table[b, used[b]:] = fill if fill is not None else free[torch.arange(rest) % len(free)].int()
        if used[b]:
            for pool, x in zip(pools, (k, v)):
                pool[ids.cuda()] = x[b, :, :used[b] * page_size].reshape(Hkv, used[b], page_size, D).permute(1, 2, 0, 3)
    return pools[0], pools[1], table.cuda()


def _call(q, kp, vp, table, o, lse, causal, splits, lq, lk):
    flash_attn.fmha_fwd(q, kp, vp, o, lse=lse, causal=causal, num_splits=splits, seqlens_q=lq, seqlens_k=lk,
                        block_table=table)


def _guarded_call(fn, q):
    obuf, o = _guarded(tuple(q.shape), torch.float16)
    lbuf, lse = _guarded(tuple(q.shape[:3]), torch.float32)
    torch.cuda.synchronize()
    n0 = _capi.launch_count()
    fn(o, lse)
    n = _capi.launch_count() - n0
    torch.cuda.synchronize()
    _assert_margins(obuf, "O")
    _assert_margins(lbuf, "lse")
    return o, lse, n


def _run(q, kp, vp, table, causal, splits, lq, lk):
    return _guarded_call(lambda o, lse: _call(q, kp, vp, table, o, lse, causal, splits, lq, lk), q)


def _run_seqlens(q, k, v, causal, splits, lq, lk):
    return _guarded_call(lambda o, lse: flash_attn.fmha_fwd(q, k, v, o, lse=lse, causal=causal, num_splits=splits,
                                                            seqlens_q=lq, seqlens_k=lk), q)[:2]


def _same(a, b):
    return torch.equal(a.nan_to_num(1.0), b.nan_to_num(1.0)) and torch.equal(a.isnan(), b.isnan())


def _check(key, got, want, bound, empty, what):
    for name, g, w, b in zip(("O", "lse"), got, want, bound):
        assert not bool(torch.isnan(g).any()), f"{what} {name}: NaN"
        if bool(empty.any()):
            assert bool((g[empty] == (-math.inf if name == "lse" else 0)).all()), f"{what} {name}: empty row"
        ne = ~empty
        err = (g.double()[ne] - w[ne]).abs()
        if err.numel() == 0:
            continue
        ratio = torch.nan_to_num(err / b[ne], nan=float("inf")).max().item()
        _ratios[(key, name)] = max(_ratios[(key, name)], ratio)
        assert bool((err <= b[ne]).all()), f"{what} {name}: |err|/bound {ratio:.3g}"


def _check_fp64(key, o, lse, q0, k0, v0, causal, splits, lq, lk, D, exact, what):
    sc, poly = R.kernel_scale(D), D <= 128
    if splits > 1:
        parts = S.part_references(q0, k0, v0, sc, causal, splits, lq, lk, exact)
        want_o, want_l, empty, ob, lb = SR.combine_bound(parts, poly)
    else:
        ref = S.reference(q0, k0, v0, sc, causal, lq, lk, exact)
        _, ob = R.o_bound(ref, poly)
        want_o, want_l, empty, lb = ref["o"], ref["lse"], ref["empty"], R.lse_bound(ref, poly)
    _check(key, (o, lse), (want_o, want_l), (ob, lb), empty, what)


@pytest.mark.parametrize("i", range(len(P.CASES_BY_SHAPE)),
                         ids=lambda i: f"case{i}-D{P.CASES_BY_SHAPE[i].D}-page{P.CASES_BY_SHAPE[i].page_size}")
def test_case(i):
    c = P.CASES_BY_SHAPE[i]
    B, Nk = len(c.lq), c.page_size * c.max_pages
    key, launches = P.path(B, c.H, c.Hkv, c.Nq, c.page_size, c.max_pages, c.D, c.causal, c.splits)
    lq, lk = _lens(c.lq), _lens(c.lk)
    for j, gen in enumerate(c.gens):
        poison = _POISON[(i + j) % len(_POISON)]
        what = (f"{label(key)}: H{c.H} Hkv{c.Hkv} Nq{c.Nq} page{c.page_size}x{c.max_pages} D{c.D} splits={c.splits} "
                f"{gen} pad={poison}")
        q0, k0, v0 = _inputs(gen, B, c.H, c.Hkv, c.Nq, Nk, c.D, None, seed=7919 * i + j)
        q, k, v = _poison(q0, k0, v0, c.lq, c.lk, poison)
        kp, vp, table = paginate(k, v, c.lk, c.page_size, c.max_pages, poison, seed=31 * i + j)
        kc, vc, tc, qc = kp.clone(), vp.clone(), table.clone(), q.clone()
        o, lse, n = _run(q, kp, vp, table, c.causal, c.splits, lq, lk)
        assert n == launches, f"{what}: {n} launches, the path has {launches}"
        assert _same(kp, kc) and _same(vp, vc) and torch.equal(table, tc) and _same(q, qc), what + ": an input changed"
        so, sl = _run_seqlens(q, k, v, c.causal, c.splits, lq, lk)
        assert torch.equal(o, so) and torch.equal(lse, sl), what + ": not bitwise the seqlens call on the padded cache"
        _check_fp64(key, o, lse, q0, k0, v0, c.causal, c.splits, c.lq, c.lk, c.D, M.exact_scores(gen), what)


# ------------------------------------------------------------------ shared pages, long sequences, graphs, SDPA
@pytest.mark.parametrize("splits", [1, 3])
def test_shared_pages(splits):
    """Sequences 0 and 1 share their first pages (a common prefix); sequence 1's own copies of them are poisoned."""
    B, H, Hkv, Nq, ps, maxp, D = 3, 8, 2, 5, 16, 40, 128
    lq, lk = [5, 5, 3], [300, 450, 77]
    q0, k0, v0 = _inputs("randn", B, H, Hkv, Nq, ps * maxp, D, None, seed=3)
    shared = 7   # pages
    k0[1, :, :shared * ps] = k0[0, :, :shared * ps]
    v0[1, :, :shared * ps] = v0[0, :, :shared * ps]
    q, k, v = _poison(q0, k0, v0, lq, lk, float("nan"))
    kp, vp, table = paginate(k, v, lk, ps, maxp, float("nan"), seed=4)
    own = table[1, :shared].long()
    kp[own] = float("nan")
    vp[own] = float("nan")
    table[1, :shared] = table[0, :shared]
    o, lse, _ = _run(q, kp, vp, table, False, splits, _lens(lq), _lens(lk))
    so, sl = _run_seqlens(q, k, v, False, splits, _lens(lq), _lens(lk))
    assert torch.equal(o, so) and torch.equal(lse, sl)
    key = P.path(B, H, Hkv, Nq, ps, maxp, D, False, splits)[0]
    _check_fp64(key, o, lse, q0, k0, v0, False, splits, lq, lk, D, False, "shared pages")


def test_long_sequence_among_short_ones():
    """One 65536-key sequence in 16-key pages (4096 table entries) in a decode batch, split automatically."""
    B, H, Hkv, Nq, ps, maxp, D = 4, 8, 2, 1, 16, 4096, 128
    lens_k = [65536, 3, 0, 700]
    q, k, v = _inputs("randn", B, H, Hkv, Nq, ps * maxp, D, None, seed=13)
    q, k, v = _poison(q, k, v, [1] * B, lens_k, float("nan"))
    kp, vp, table = paginate(k, v, lens_k, ps, maxp, float("nan"), seed=14)
    splits = _capi.lib().b200_fmha_fwd_f16_gqa_splits(B, H, Hkv, Nq, ps * maxp, D)
    assert splits > 1
    lq, lk = _lens([1] * B), _lens(lens_k)
    o, lse, n = _run(q, kp, vp, table, False, 0, lq, lk)
    assert n == 2
    so, sl = _run_seqlens(q, k, v, False, 0, lq, lk)
    assert torch.equal(o, so) and torch.equal(lse, sl)
    key = P.path(B, H, Hkv, Nq, ps, maxp, D, False, splits)[0]
    _check_fp64(key, o, lse, q.clone(), k.nan_to_num(0.0), v.nan_to_num(0.0), False, splits, [1] * B, lens_k, D, False,
                "long sequence")


@pytest.mark.parametrize("splits", [1, 4], ids=["unsplit", "split"])
def test_graph_replay_with_new_tables_and_side_stream(splits):
    """A captured call replays with the tables and lengths written into the same tensors afterwards, bit for bit the
    eager call; a call on a side stream equals the eager one."""
    B, H, Hkv, Nq, ps, maxp, D = 6, 16, 4, 1, 16, 128, 128
    q, k, v = _inputs("randn", B, H, Hkv, Nq, ps * maxp, D, None, seed=11)
    kp, vp, table = paginate(k, v, [ps * maxp] * B, ps, maxp, float("nan"), seed=12)
    lq, lk = _lens([1] * B), _lens([5, 2048, 64, 0, 1000, 129])
    o, lse = torch.empty_like(q), torch.empty(q.shape[:3], device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            _call(q, kp, vp, table, o, lse, False, splits, lq, lk)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    eo, el, _ = _run(q, kp, vp, table, False, splits, lq, lk)
    assert torch.equal(o, eo) and torch.equal(lse, el), "side stream differs from eager"
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        _call(q, kp, vp, table, o, lse, False, splits, lq, lk)
    base = table.clone()
    for shift, new_k in ((1, [2048, 1, 0, 700, 63, 65]), (3, [100, 200, 300, 400, 500, 600])):
        table.copy_(base.roll(shift, 0))   # sequence b now reads the pages of sequence b - shift
        lk.copy_(_lens(new_k))
        graph.replay()
        torch.cuda.synchronize()
        eo, el, _ = _run(q, kp, vp, table, False, splits, lq, lk)
        assert torch.equal(o, eo) and torch.equal(lse, el), f"graph replay with table shift {shift} differs from eager"
        assert not torch.equal(table, base)


def _bench_lengths(index):
    """The seeded length draws of tools/bench_attn_paged.py (and bench_attn_seqlens.py) up to shape `index`."""
    rng = np.random.default_rng(0)
    for name, B, _, _, _, _, _, _, (lo, hi) in BENCH_SHAPES[:index + 1]:
        lk = [int(x) for x in rng.integers(lo, hi + 1, size=B)]
    return lk


def _sampled_rows(lq, lk, D, causal):
    if lq <= 16:
        return list(range(lq))
    kbn, per = M.kernel_shape(D)
    rows = {0, 63, 64, lq - 1, lq - 2}
    rows |= {i for i in range(lq) if causal and (i + lk - lq) % kbn in (0, kbn - 1)}
    return sorted(r for r in rows if 0 <= r < lq)[:48]


@pytest.mark.parametrize("index", range(len(BENCH_SHAPES)), ids=lambda i: BENCH_SHAPES[i][0].replace(" ", "-") + str(i))
def test_benchmarked_shape(index):
    """Every shape of tools/bench_attn_paged.py at full size and both page sizes: bit for bit gather + seqlens, and
    sampled rows of three sequences within the fp64 bound."""
    name, B, H, Hkv, Nq, Nk, D, causal, _ = BENCH_SHAPES[index]
    lk = _bench_lengths(index)
    lq = lk if causal else [Nq] * B
    g = torch.Generator(device="cuda").manual_seed(100 + index)
    q = torch.randn(B, H, Nq, D, device="cuda", generator=g).half()
    k = torch.randn(B, Hkv, Nk, D, device="cuda", generator=g).half()
    v = torch.randn(B, Hkv, Nk, D, device="cuda", generator=g).half()
    tq, tk = _lens(lq), _lens(lk)
    splits = _capi.lib().b200_fmha_fwd_f16_gqa_splits(B, H, Hkv, Nq, Nk, D)
    sc, poly = R.kernel_scale(D), True
    for ps in BENCH_PAGE_SIZES:
        kp, vp, table = paginate(k, v, lk, ps, Nk // ps, float("nan"), seed=ps + index, pad=-1)
        o, lse, n = _run(q, kp, vp, table, causal, 0, tq, tk)
        assert n == 1 + (splits > 1)
        kg, vg = P.gather(kp, table, lk, Nk), P.gather(vp, table, lk, Nk)
        so, sl = _run_seqlens(q, kg, vg, causal, 0, tq, tk)
        assert torch.equal(o, so) and torch.equal(lse, sl), f"{name} page {ps}: not bitwise gather + seqlens"
        key = P.path(B, H, Hkv, Nq, ps, Nk // ps, D, causal, splits)[0]
        for b in sorted({int(np.argmin(lk)), int(np.argmax(lk)), B // 2}):
            what = f"{name} page {ps} sequence {b} (Lq {lq[b]}, Lk {lk[b]})"
            qb, kb, vb = q[b:b + 1], kg[b:b + 1, :, :lk[b]], vg[b:b + 1, :, :lk[b]]
            if splits > 1:
                _check_fp64(key, o[b:b + 1], lse[b:b + 1], qb, kb, vb, causal, splits, [lq[b]], [lk[b]], D, False, what)
                continue
            r = torch.tensor(_sampled_rows(lq[b], lk[b], D, causal), device="cuda")
            i, j = r[:, None], torch.arange(lk[b], device="cuda")[None, :]
            vis = (j <= i + (lk[b] - lq[b])) if causal else torch.ones_like(i * j, dtype=torch.bool)
            G = H // Hkv
            ref = SR.masked_reference(qb[:, :, r], SR.expand(kb, G), SR.expand(vb, G), sc, vis[None, None])
            _, ob = R.o_bound(ref, poly)
            _check(key, (o[b:b + 1, :, r], lse[b:b + 1, :, r]), (ref["o"], ref["lse"]), (ob, R.lse_bound(ref, poly)),
                   ref["empty"], what)
        del kp, vp, kg, vg
        torch.cuda.empty_cache()


def test_sdpa_with_an_explicit_mask():
    B, H, Hkv, Nq, ps, maxp, D = 3, 8, 2, 40, 16, 32, 64
    q, k, v = _inputs("randn", B, H, Hkv, Nq, ps * maxp, D, None, seed=17)
    lq, lk = [40, 7, 1], [512, 300, 9]
    kp, vp, table = paginate(k, v, lk, ps, maxp, float("nan"), seed=18)
    o, _, _ = _run(q, kp, vp, table, True, 1, _lens(lq), _lens(lk))
    kg, vg = P.gather(kp, table, lk, ps * maxp), P.gather(vp, table, lk, ps * maxp)
    vis = torch.from_numpy(np.stack([S.visible(Nq, ps * maxp, lq[b], lk[b], True) for b in range(B)])[:, None]).cuda()
    ref = F.scaled_dot_product_attention(q, kg, vg, attn_mask=vis, enable_gqa=True)
    for b in range(B):
        err = (o[b, :, :lq[b]].float() - ref[b, :, :lq[b]].float()).abs().max().item()
        assert err < 2e-3, (b, err)
        assert bool((o[b, :, lq[b]:] == 0).all())


# ------------------------------------------------------------------ kernel names
# torch.profiler runs in a child process, all cases in one session (test_attn_seqlens_gpu._kernels_per_call); this
# process never starts it.  On an H100, in one process, sessions that came after an earlier session followed by many
# launches recorded some or none of their kernels.
def _profile_all_cases():
    """Child process: the CUDA kernel names of every case, as one JSON line on stdout."""
    import json
    fns = []
    for i, c in enumerate(P.CASES_BY_SHAPE):
        q, k, v = _inputs("randn", len(c.lq), c.H, c.Hkv, c.Nq, c.page_size * c.max_pages, c.D, None, seed=i)
        kp, vp, table = paginate(k, v, c.lk, c.page_size, c.max_pages, 0.0, seed=i)
        lq, lk, o = _lens(c.lq), _lens(c.lk), torch.empty_like(q)
        fns.append(lambda a=(q, kp, vp, table, o, None, c.causal, c.splits, lq, lk): _call(*a))
    print("KERNEL_NAMES " + json.dumps(_kernels_per_call(fns)))


@pytest.fixture(scope="module")
def profiled_names():
    return profiled_names_of("test_attn_paged_gpu")


@pytest.mark.parametrize("i", range(len(P.CASES_BY_SHAPE)),
                         ids=lambda i: f"case{i}-D{P.CASES_BY_SHAPE[i].D}-page{P.CASES_BY_SHAPE[i].page_size}")
def test_kernel_names(profiled_names, i):
    c = P.CASES_BY_SHAPE[i]
    key, _ = P.path(len(c.lq), c.H, c.Hkv, c.Nq, c.page_size, c.max_pages, c.D, c.causal, c.splits)
    what = f"{label(key)}: H{c.H} Hkv{c.Hkv} Nq{c.Nq} page{c.page_size}x{c.max_pages} D{c.D} splits={c.splits}"
    names = profiled_names[i] if i < len(profiled_names) else []
    assert names, what + ": the profiler recorded no kernel"
    assert P.parse_instantiations(names) == [P.instantiation(key)], f"{what}: ran {names}"
    assert not S.parse_instantiations(names), f"{what}: ran {names}"
    assert sum("attn_combine_kernel" in s for s in names) == int(key[4]), f"{what}: ran {names}"
