"""fp8 (e4m3) K/V attention (flash_attn.fmha_fwd with float8_e4m3fn K and V: b200_fmha_fwd_{f16,bf16}_fp8kv_{seqlens,
paged}) on the GPU, over every path of attn_fp8kv_ref.CASES for fp16 and bf16 Q/O.

Every case fills the valid V rows with all 254 finite e4m3 codes (test_all_codes also K), poisons what lies past the
lengths (K / V codes NaN 0x7F / 0xFF or +-448, unused pages alike, table padding -1, INT_MIN or ids of poisoned pages,
Q rows >= Lq_b NaN) and puts O and lse inside NaN guard bands.  Checked:
  * bit for bit the T call (b200_fmha_fwd_{f16,bf16}_seqlens / _paged, also for a dense fp8 call) on K.to(T), V.to(T)
    with v_scale = 1 and scale = fp32(scale * k_scale);
  * against fp64 on the dequantised K and V within attn_fp8kv_ref's bound, for scales 1, powers of two, 0.37 and large
    ones; padded rows and rows without a key exactly O = 0, lse = -inf; the inputs, the pool and the table unchanged;
  * _capi.launch_count() up by 1 unsplit, 2 split; kernel names under torch.profiler in a child process only (this
    process never starts the profiler: the fp16 modules that sort after this one rely on the first sessions).
Then CUDA graph replay with new lengths and tables and a side stream, and every shape of tools/bench_attn_fp8kv.py at
full size.  The largest |err| / bound per path is printed at the end of the module (pytest -s).
"""
import collections
import json
import math
import os
import subprocess
import sys
import time
from pathlib import Path

import numpy as np
import pytest
import torch

import attn_fp8kv_ref as F
import attn_mask_ref as M
import attn_paged_ref as P
import attn_ref as R
import attn_seqlens_ref as S
import attn_split_ref as SR
from leetcuda_b200 import _capi, flash_attn
from test_attn_gqa_gpu import _inputs
from test_attn_numerics_gpu import MARGIN, SENT32, _assert_margins
from test_attn_seqlens_gpu import _kernels_per_call, _lens

pytestmark = pytest.mark.gpu

# the shapes of tools/bench_attn_fp8kv.py (test_attn_fp8kv_coverage checks that they agree):
# (name, B, H, Hkv, Nq, Nk, D, causal, kind, page_size)
BENCH_SHAPES = [
    ("dense decode", 8, 32, 8, 1, 8192, 128, False, "dense", None),
    ("seqlens decode", 32, 32, 8, 1, 8192, 128, False, "seqlens", None),
    ("paged decode p16", 32, 32, 8, 1, 8192, 128, False, "paged", 16),
    ("paged decode p256", 32, 32, 8, 1, 8192, 128, False, "paged", 256),
    ("long decode", 4, 64, 8, 1, 32768, 128, False, "dense", None),
    ("paged causal prefill", 8, 32, 8, 4096, 4096, 128, True, "paged", 256),
]
BENCH_LK_RANGE = (256, 8192)
_ratios = collections.defaultdict(float)
_KV_POISON = (0x7F, 0xFF, 0x7E, 0xFE)   # NaN, NaN, 448, -448
SENT16 = {torch.float16: 0x7E01, torch.bfloat16: 0x7FC1}   # NaNs the kernel never writes
_codes_seen = set()


def label(key):
    T, kind, ds, bn, wg, causal, split, tiling = key[:8]
    flags = [f for f, on in (("causal", causal), ("split", split)) if on]
    return f"{T} {kind} <{','.join([str(ds), str(bn), str(wg)] + flags)}> {tiling}" + (f" page{key[8]}" if len(key) > 8
                                                                                       else "")


@pytest.fixture(scope="module", autouse=True)
def _report():
    t0 = time.time()
    yield
    if _ratios:
        print("\nlargest |err| / bound per path (attn_fp8kv_ref.o_bound / lse_bound / combine_bound):")
        for key in sorted({k for k, _ in _ratios}, key=str):
            print(f"  {label(key):<52} O {_ratios[(key, 'O')]:.3f}  lse {_ratios[(key, 'lse')]:.3f}")
    print(f"module time {time.time() - t0:.1f} s")


# ------------------------------------------------------------------ helpers
def _guarded(shape, dtype):
    n = int(np.prod(shape))
    buf = torch.empty(n + 2 * MARGIN, dtype=dtype, device="cuda")
    if dtype == torch.float32:
        buf.view(torch.int32).fill_(SENT32)
    else:
        buf.view(torch.int16).fill_(SENT16[dtype])
    return buf, buf[MARGIN:MARGIN + n].view(shape)


def _margins_ok(buf, what):
    if buf.dtype == torch.float32:
        _assert_margins(buf, what)
        return
    bits = buf.view(torch.int16)
    assert bool((bits[:MARGIN] == SENT16[buf.dtype]).all()), f"{what}: store before the output"
    assert bool((bits[-MARGIN:] == SENT16[buf.dtype]).all()), f"{what}: store past the output"


def _guarded_call(fn, q):
    obuf, o = _guarded(tuple(q.shape), q.dtype)
    lbuf, lse = _guarded(tuple(q.shape[:3]), torch.float32)
    torch.cuda.synchronize()
    n0 = _capi.launch_count()
    fn(o, lse)
    n = _capi.launch_count() - n0
    torch.cuda.synchronize()
    _margins_ok(obuf, "O")
    _margins_ok(lbuf, "lse")
    return o, lse, n


def _fp8(codes):
    return codes.view(torch.float8_e4m3fn)


def _fp8_call(q, k8, v8, causal, splits, lq, lk, table, ks, vs):
    kw = dict(causal=causal, num_splits=splits, seqlens_q=lq, seqlens_k=lk, k_scale=ks, v_scale=vs)
    if table is not None:
        kw["block_table"] = table
    return _guarded_call(lambda o, lse: flash_attn.fmha_fwd(q, k8, v8, o, lse=lse, **kw), q)


def _t_call(q, k8, v8, causal, splits, lq, lk, table, scale):
    """The T entry (seqlens or paged, never the dense fp16 kernel) on K, V widened to T, with the folded scale."""
    T = q.dtype
    kt, vt = k8.to(T), v8.to(T)
    o, lse = torch.empty_like(q), torch.empty(q.shape[:3], device="cuda")
    B, H, Nq, D = q.shape
    pre = "b200_fmha_fwd_bf16" if T == torch.bfloat16 else "b200_fmha_fwd_f16"
    lens = [None if lq is None else lq.data_ptr(), None if lk is None else lk.data_ptr()]
    if table is None:
        args = [q.data_ptr(), kt.data_ptr(), vt.data_ptr(), o.data_ptr(), lse.data_ptr(), *lens, B, H, kt.shape[1], Nq,
                kt.shape[2], D, int(causal), splits, scale]
        fn = getattr(_capi.lib(), pre + "_seqlens")
    else:
        args = [q.data_ptr(), kt.data_ptr(), vt.data_ptr(), o.data_ptr(), lse.data_ptr(), table.data_ptr(), *lens, B, H,
                kt.shape[2], Nq, kt.shape[0], kt.shape[1], table.shape[1], D, int(causal), splits, scale]
        fn = getattr(_capi.lib(), pre + "_paged")
    flash_attn._call_on_device(fn, args, q.device.index)
    torch.cuda.synchronize()
    return o, lse


def _fold(scale, ks):
    return float(np.float32(np.float32(scale) * np.float32(ks)))


def _sweep(shape, seed):
    """uint8 codes of `shape` cycling through a random permutation of the 254 finite codes."""
    codes = F.finite_codes()[torch.randperm(254, generator=torch.Generator().manual_seed(seed))]
    n = int(np.prod(shape))
    return codes.repeat(-(-n // 254))[:n].view(shape).cuda()


def _make(gen, T, B, H, Hkv, Nq, Nk, D, lq, lk, seed, k_sweep=False):
    """q (T, rows >= Lq_b NaN) and clean uint8 K / V codes (V: every finite code over the valid rows; K: the generator's
    values quantised, or every code with k_sweep), and the poisoned copies."""
    q0, k0, _ = _inputs(gen, B, H, Hkv, Nq, Nk, D, None, seed=seed)
    q0 = q0.to(F.TORCH[T])
    k = _sweep(k0.shape, seed + 1) if k_sweep else F.quantise(k0, 1.0).view(torch.uint8)
    v = _sweep(k0.shape, seed + 2)
    q, kp, vp = q0.clone(), k.clone(), v.clone()
    for b in range(B):
        q[b, :, lq[b]:] = float("nan")
        kp[b, :, lk[b]:] = _KV_POISON[(seed + b) % 4]
        vp[b, :, lk[b]:] = _KV_POISON[(seed + b + 1) % 4]
        _codes_seen.update(v[b, :, :lk[b]].unique().tolist())
        if k_sweep:
            _codes_seen.update(k[b, :, :lk[b]].unique().tolist())
    return q0, k, v, q, kp, vp


def paginate(k, v, lk, page_size, max_pages, poison, pad, seed):
    """uint8 pools [num_pages, page_size, Hkv, D] holding k, v in randomly placed pages, unused pages `poison`, and the
    table [B, max_pages] padded past each sequence's pages with `pad`: an int, or "poisoned" for ids of unused pages."""
    B, Hkv, _, D = k.shape
    used = [-(-x // page_size) for x in lk]
    n_used = sum(used)
    num_pages = n_used + max(4, n_used // 4)
    perm = torch.randperm(num_pages, generator=torch.Generator().manual_seed(seed))
    pools = [torch.full((num_pages, page_size, Hkv, D), poison, dtype=torch.uint8, device="cuda") for _ in range(2)]
    spare = perm[n_used:]
    table = torch.empty((B, max_pages), dtype=torch.int32)
    for b in range(B):
        table[b] = spare[torch.arange(max_pages) % len(spare)].int() if pad == "poisoned" else pad
    n = 0
    for b in range(B):
        ids = perm[n:n + used[b]]
        n += used[b]
        table[b, :used[b]] = ids.int()
        if used[b]:
            for pool, x in zip(pools, (k, v)):
                pool[ids.cuda()] = x[b, :, :used[b] * page_size].reshape(Hkv, used[b], page_size, D).permute(1, 2, 0, 3)
    return pools[0], pools[1], table.cuda()


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


def _check_fp64(key, T, o, lse, q0, k, v, causal, splits, lq, lk, D, scale, ks, vs, what):
    """k, v: clean uint8 codes.  The truth is vs * attention(scale * ks) on the code values; the bound's reference runs
    at the kernel's folded scale."""
    kd, vd = F.decode(k), F.decode(v)
    sc = _fold(scale, ks)
    poly = D <= 128
    G = q0.shape[1] // k.shape[1]
    xmax = F.score_max(q0, SR.expand(kd, G), sc)
    truth = S.reference(q0, kd, vd, scale * ks, causal, lq, lk)
    if splits > 1:
        parts = S.part_references(q0, kd, vd, sc, causal, splits, lq, lk)
        vmax = SR.expand(vd.abs().amax(-2, keepdim=True), G)
        _, _, empty, ob, lb = F.combine_bound(parts, poly, T, vs, xmax, vmax)
    else:
        ref = S.reference(q0, kd, vd, sc, causal, lq, lk)
        empty, ob, lb = ref["empty"], F.o_bound(ref, poly, T, vs, xmax), F.lse_bound(ref, poly, xmax)
    assert torch.equal(empty, truth["empty"])
    _check(key, (o, lse), (vs * truth["o"], truth["lse"]), (ob, lb), empty, what)


def _resolved(splits, B, H, Hkv, Nq, Nk, D):
    return splits if splits else _capi.lib().b200_fmha_fwd_f16_gqa_splits(B, H, Hkv, Nq, Nk, D)


# ------------------------------------------------------------------ the case table
def _run_case(i, k_sweep=False, scales=None):
    T, kind, c = F.CASES[i]
    dense = kind == "dense"
    B = 2 if dense else len(c.lq)
    Nk = c.page_size * c.max_pages if kind == "paged" else c.Nk
    lq_l, lk_l = ([c.Nq] * B, [c.Nk] * B) if dense else (c.lq, c.lk)
    lqc, lkc = S.clamp(lq_l, c.Nq), S.clamp(lk_l, Nk)
    splits = _resolved(c.splits, B, c.H, c.Hkv, c.Nq, Nk, c.D)
    key, launches = F.path(kind, T, B, c.H, c.Hkv, c.Nq, Nk, c.D, c.causal, c.splits, getattr(c, "page_size", None))
    assert key == F.case_key(T, kind, c) or c.splits == 0
    for j, gen in enumerate(c.gens):
        seed = 7919 * i + 31 * j
        q0, k, v, q, kp, vp = _make(gen, T, B, c.H, c.Hkv, c.Nq, Nk, c.D, lqc, lkc, seed, k_sweep)
        lq, lk = (None, None) if dense else (_lens(c.lq), _lens(c.lk))
        table = None
        if kind == "paged":
            pad = (-1, -2 ** 31, "poisoned")[(i + j) % 3]
            kp, vp, table = paginate(kp, vp, lkc, c.page_size, c.max_pages, _KV_POISON[(i + j) % 4], pad, seed)
        saved = [x.clone() for x in (q, kp, vp) + (() if table is None else (table,))]
        scale = R.kernel_scale(c.D)
        what = f"{label(key)}: H{c.H} Hkv{c.Hkv} Nq{c.Nq} Nk{Nk} D{c.D} splits={c.splits} {gen}"
        # v_scale = 1: bit for bit the T call with the folded scale
        ks = (1.0, 0.5, 0.37)[(i + j) % 3]
        o, lse, n = _fp8_call(q, _fp8(kp), _fp8(vp), c.causal, c.splits, lq, lk, table, ks, 1.0)
        assert n == launches, f"{what}: {n} launches, the path has {launches}"
        eo, el = _t_call(q, _fp8(kp), _fp8(vp), c.causal, c.splits, lq, lk, table, _fold(scale, ks))
        assert torch.equal(o, eo) and torch.equal(lse, el), f"{what}: not bitwise the T call with k_scale={ks} folded"
        _check_fp64(key, T, o, lse, q0, k, v, c.causal, splits, lqc, lkc, c.D, scale, ks, 1.0, what + f" ks={ks}")
        # scales != 1 against fp64
        for sc_ in scales or [F.SCALES[1 + (i + j) % (len(F.SCALES) - 1)]]:
            o, lse, n = _fp8_call(q, _fp8(kp), _fp8(vp), c.causal, c.splits, lq, lk, table, sc_.k, sc_.v)
            assert n == launches
            _check_fp64(key, T, o, lse, q0, k, v, c.causal, splits, lqc, lkc, c.D, scale, sc_.k, sc_.v,
                        what + f" scales={tuple(sc_)}")
        for x, y in zip((q, kp, vp) + (() if table is None else (table,)), saved):
            assert torch.equal(x.view(torch.uint8) if x.dtype != torch.int32 else x,
                               y.view(torch.uint8) if y.dtype != torch.int32 else y), what + ": an input changed"


@pytest.mark.parametrize("i", range(len(F.CASES)), ids=lambda i: f"{F.CASES[i][0]}-{F.CASES[i][1]}{i}-D{F.CASES[i][2].D}")
def test_case(i):
    _run_case(i)


def _first(T, kind, causal, split):
    return next(i for i, (t, k, c) in enumerate(F.CASES)
                if t == T and k == kind and c.causal == causal and (c.splits != 1) == split and c.D <= 128)


@pytest.mark.parametrize("T", F.TYPES)
@pytest.mark.parametrize("kind", ["seqlens", "paged"])
def test_all_codes(T, kind):
    """K and V both sweep every finite code (subnormals, +-448 and -0 among them) under every scale of the table."""
    for causal, split in ((False, False), (True, True)):
        _run_case(_first(T, kind, causal, split), k_sweep=True, scales=F.SCALES[1:])


def test_cases_held_every_finite_code():
    if len(_codes_seen) < 254:
        pytest.skip("runs after the case tests")
    assert _codes_seen == set(F.finite_codes().tolist())
    assert {0x00, 0x80, 0x01, 0x81, 0x7E, 0xFE} <= _codes_seen   # 0, -0, smallest subnormals, +-448


# ------------------------------------------------------------------ graphs and streams
@pytest.mark.parametrize("T", F.TYPES)
@pytest.mark.parametrize("splits", [1, 4], ids=["unsplit", "split"])
def test_graph_replay_with_new_lengths_and_tables(T, splits):
    B, H, Hkv, Nq, ps, maxp, D = 6, 16, 4, 1, 16, 128, 128
    full = [ps * maxp] * B
    q0, k, v, _, _, _ = _make("randn", T, B, H, Hkv, Nq, ps * maxp, D, [Nq] * B, full, seed=11)
    kp, vp, table = paginate(k, v, full, ps, maxp, 0x7F, -1, seed=12)
    lq, lk = _lens([1] * B), _lens([5, 2048, 64, 0, 1000, 129])
    o, lse = torch.empty_like(q0), torch.empty(q0.shape[:3], device="cuda")
    call = lambda: flash_attn.fmha_fwd(q0, _fp8(kp), _fp8(vp), o, lse=lse, num_splits=splits, seqlens_q=lq,
                                       seqlens_k=lk, block_table=table, k_scale=0.37, v_scale=2.0)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        call()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    eo, el, _ = _fp8_call(q0, _fp8(kp), _fp8(vp), False, splits, lq, lk, table, 0.37, 2.0)
    assert torch.equal(o, eo) and torch.equal(lse, el), "the call on a side stream differs from the current stream's"
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        call()
    base = table.clone()
    for shift, new_k in ((1, [2048, 1, 0, 700, 63, 65]), (3, [100, 200, 300, 400, 500, 600])):
        table.copy_(base.roll(shift, 0))
        lk.copy_(_lens(new_k))
        graph.replay()
        torch.cuda.synchronize()
        eo, el, _ = _fp8_call(q0, _fp8(kp), _fp8(vp), False, splits, lq, lk, table, 0.37, 2.0)
        assert torch.equal(o, eo) and torch.equal(lse, el), f"graph replay with table shift {shift} differs from eager"


# ------------------------------------------------------------------ the benchmarked shapes
def bench_lengths(index):
    """The seeded length draws of tools/bench_attn_fp8kv.py for shape `index`."""
    name, B, _, _, Nq, Nk, _, causal, kind, _ = BENCH_SHAPES[index]
    if kind == "dense" or causal:
        return [Nk] * B
    rng = np.random.default_rng(index)
    return [int(x) for x in rng.integers(BENCH_LK_RANGE[0], BENCH_LK_RANGE[1] + 1, size=B)]


def _sampled_rows(lq, lk, D, causal):
    if lq <= 16:
        return list(range(lq))
    kbn, _ = M.kernel_shape(D)
    rows = {0, 63, 64, 127, 128, lq - 1, lq - 2}
    rows |= {i for i in range(lq) if causal and (i + lk - lq) % kbn in (0, kbn - 1)}
    return sorted(r for r in rows if 0 <= r < lq)[:48]


@pytest.mark.parametrize("T", F.TYPES)
@pytest.mark.parametrize("index", range(len(BENCH_SHAPES)), ids=lambda i: BENCH_SHAPES[i][0].replace(" ", "-"))
def test_benchmarked_shape(index, T):
    """Every shape of tools/bench_attn_fp8kv.py at full size with k_scale 0.37, v_scale 2: bit for bit the T call at
    v_scale 1, sampled rows of three sequences within the fp64 bound (whole rows when the call splits)."""
    name, B, H, Hkv, Nq, Nk, D, causal, kind, ps = BENCH_SHAPES[index]
    lk_l = bench_lengths(index)
    lq_l = [Nq] * B
    g = torch.Generator(device="cuda").manual_seed(300 + index)
    q = torch.randn(B, H, Nq, D, device="cuda", generator=g).to(F.TORCH[T])
    k = F.quantise(torch.randn(B, Hkv, Nk, D, device="cuda", generator=g), 1.0).view(torch.uint8)
    v = _sweep((B, Hkv, Nk, D), 17 + index)
    lq, lk = (None, None) if kind == "dense" else (_lens(lq_l), _lens(lk_l))
    table = None
    if kind == "paged":
        k, v, table = paginate(k, v, lk_l, ps, Nk // ps, 0xFF, -1, seed=index)
    splits = 0 if Nq == 1 else 1
    resolved = _resolved(splits, B, H, Hkv, Nq, Nk, D)
    ks, vs = 0.37, 2.0
    o, lse, n = _fp8_call(q, _fp8(k), _fp8(v), causal, splits, lq, lk, table, 1.0 / 64, 1.0)
    assert n == 1 + (resolved > 1)
    eo, el = _t_call(q, _fp8(k), _fp8(v), causal, splits, lq, lk, table, _fold(R.kernel_scale(D), 1.0 / 64))
    assert torch.equal(o, eo) and torch.equal(lse, el), f"{name}: not bitwise the T call"
    o, lse, _ = _fp8_call(q, _fp8(k), _fp8(v), causal, splits, lq, lk, table, ks, vs)
    if table is not None:
        k = P.gather(k, table, lk_l, Nk)
        v = P.gather(v, table, lk_l, Nk)
        del table
    key = F.path("paged" if kind == "paged" else "seqlens", T, B, H, Hkv, Nq, Nk, D, causal, resolved, ps)[0]
    scale, poly, G = R.kernel_scale(D), D <= 128, H // Hkv
    sc = _fold(scale, ks)
    for b in sorted({int(np.argmin(lk_l)), int(np.argmax(lk_l)), B // 2}):
        what = f"{name} {T} sequence {b} (Lq {lq_l[b]}, Lk {lk_l[b]})"
        qb, kb, vb = q[b:b + 1], F.decode(k[b:b + 1, :, :lk_l[b]]), F.decode(v[b:b + 1, :, :lk_l[b]])
        if resolved > 1:
            _check_fp64(key, T, o[b:b + 1], lse[b:b + 1], qb, k[b:b + 1, :, :lk_l[b]].contiguous(),
                        v[b:b + 1, :, :lk_l[b]].contiguous(), causal, resolved, [lq_l[b]], [lk_l[b]], D, scale, ks, vs,
                        what)
            continue
        r = torch.tensor(_sampled_rows(lq_l[b], lk_l[b], D, causal), device="cuda")
        i, j = r[:, None], torch.arange(lk_l[b], device="cuda")[None, :]
        vis = (j <= i + (lk_l[b] - lq_l[b])) if causal else torch.ones_like(i * j, dtype=torch.bool)
        kx, vx = SR.expand(kb, G), SR.expand(vb, G)
        ref = SR.masked_reference(qb[:, :, r], kx, vx, sc, vis[None, None])
        truth = SR.masked_reference(qb[:, :, r], kx, vx, scale * ks, vis[None, None])
        xmax = F.score_max(qb[:, :, r], kx, sc)
        _check(key, (o[b:b + 1, :, r], lse[b:b + 1, :, r]), (vs * truth["o"], truth["lse"]),
               (F.o_bound(ref, poly, T, vs, xmax), F.lse_bound(ref, poly, xmax)), ref["empty"], what)
    del q, k, v, o, lse
    torch.cuda.empty_cache()


# ------------------------------------------------------------------ kernel names
# torch.profiler runs in a child process, all cases in one session; the test process never starts the profiler (see
# test_attn_bf16_gpu: a session followed by many launches leaves later sessions of the process without CUDA records).
def _case_call(i):
    T, kind, c = F.CASES[i]
    dense = kind == "dense"
    B = 2 if dense else len(c.lq)
    Nk = c.page_size * c.max_pages if kind == "paged" else c.Nk
    key = F.path(kind, T, B, c.H, c.Hkv, c.Nq, Nk, c.D, c.causal,
                 _resolved(c.splits, B, c.H, c.Hkv, c.Nq, Nk, c.D), getattr(c, "page_size", None))[0]
    lqc, lkc = ([c.Nq] * B, [Nk] * B) if dense else (S.clamp(c.lq, c.Nq), S.clamp(c.lk, Nk))
    q0, k, v, _, _, _ = _make("randn", T, B, c.H, c.Hkv, c.Nq, Nk, c.D, lqc, lkc, seed=i)
    kw = dict(causal=c.causal, num_splits=c.splits, k_scale=0.5, v_scale=0.5)
    if not dense:
        kw.update(seqlens_q=_lens(c.lq), seqlens_k=_lens(c.lk))
    if kind == "paged":
        k, v, table = paginate(k, v, lkc, c.page_size, c.max_pages, 0, -1, seed=i)
        kw["block_table"] = table
    o = torch.empty_like(q0)
    fn = lambda: flash_attn.fmha_fwd(q0, _fp8(k), _fp8(v), o, **kw)
    return key, fn, f"{label(key)}: {kind} H{c.H} Hkv{c.Hkv} Nq{c.Nq} D{c.D} splits={c.splits}"


def _profile_all_cases():
    """Child process: the CUDA kernel names of every case under torch.profiler, as one JSON line on stdout."""
    fns = [_case_call(i)[1] for i in range(len(F.CASES))]
    print("KERNEL_NAMES " + json.dumps(_kernels_per_call(fns)))


@pytest.fixture(scope="module")
def profiled_names():
    tests = Path(__file__).resolve().parent
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([str(tests.parent), str(tests)]
                                                      + [p for p in [os.environ.get("PYTHONPATH")] if p]))
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [
        "-c", "import test_attn_fp8kv_gpu as T; T._profile_all_cases()"]
    r = subprocess.run(cmd, cwd=tests.parent, env=env, capture_output=True, text=True, timeout=900)
    lines = [x for x in r.stdout.splitlines() if x.startswith("KERNEL_NAMES ")]
    assert r.returncode == 0 and lines, f"profiling child failed ({r.returncode}):\n{r.stdout[-2000:]}{r.stderr[-4000:]}"
    return json.loads(lines[-1][len("KERNEL_NAMES "):])


@pytest.mark.parametrize("i", range(len(F.CASES)), ids=lambda i: f"{F.CASES[i][0]}-{F.CASES[i][1]}{i}-D{F.CASES[i][2].D}")
def test_kernel_names(profiled_names, i):
    import attn_bf16_ref as BF
    key, _, what = _case_call(i)
    names = profiled_names[i]
    assert names, what + ": the profiler recorded no kernel"
    assert F.parse_instantiations(names) == [F.instantiation(key)], f"{what}: ran {names}"
    assert not BF.parse_instantiations(names), f"{what}: ran {names}"
    assert not S.parse_instantiations(names) and not P.parse_instantiations(names), f"{what}: ran {names}"
    assert not any("attn_fwd_kernel<" in s for s in names), f"{what}: ran {names}"
    assert sum("attn_combine_kernel" in s for s in names) == int(key[6]), f"{what}: ran {names}"
