"""bf16 attention (flash_attn.fmha_fwd on bf16 tensors: b200_fmha_fwd_bf16_seqlens / _paged) on the GPU, over every path
of attn_bf16_ref.CASES.

Every case poisons what lies past the lengths (K / V rows >= Lk_b NaN, +Inf, -Inf or 65504, Q rows >= Lq_b NaN) and puts
O and lse inside guard bands.  Checked:
  * the fp64 reference of the bf16 inputs with attn_bf16_ref.o_bound / lse_bound (combine_bound when split); padded
    rows and rows without a key exactly O = 0, lse = -inf; the inputs come back unchanged;
  * paged: bit for bit the bf16 seqlens call on the gathered cache; seqlens unsplit: every sequence bit for bit the
    call on that sequence alone; dense GQA: bit for bit the call on K / V with every head repeated (num_splits=1);
  * _capi.launch_count() up by 1 unsplit, 2 split; under torch.profiler (in a child process, so that this process
    never starts the profiler) the restated bf16 kernel and no other attention kernel, the combine exactly when the
    call splits.
Then inputs outside fp16's range, CUDA graph replay with new lengths and tables, two key halves merged by
merge_attn_states in bf16, and every shape of tools/bench_attn_bf16.py at full size.  The largest |err| / bound per path
is printed at the end of the module (pytest -s).
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

import attn_bf16_ref as BF
import attn_mask_ref as M
import attn_paged_ref as P
import attn_ref as R
import attn_seqlens_ref as S
import attn_split_ref as SR
from leetcuda_b200 import _capi, flash_attn
from leetcuda_b200 import merge_attn_states as MA
from test_attn_gqa_gpu import _inputs
from test_attn_numerics_gpu import MARGIN, SENT32, _assert_margins
from test_attn_seqlens_gpu import _kernels_per_call, _lens, _poison

pytestmark = pytest.mark.gpu

# the shapes of tools/bench_attn_bf16.py (test_attn_bf16_coverage checks that they agree)
BENCH_SHAPES = [
    ("dense", 4, 32, 32, 4096, 4096, 128, False, "dense"),
    ("dense", 4, 32, 32, 4096, 4096, 128, True, "dense"),
    ("dense", 4, 32, 32, 4096, 4096, 64, False, "dense"),
    ("dense", 4, 32, 32, 4096, 4096, 64, True, "dense"),
    ("decode", 8, 32, 8, 1, 8192, 128, False, "decode"),
    ("seqlens decode", 32, 32, 8, 1, 8192, 128, False, "seqlens"),
    ("paged decode", 32, 32, 8, 1, 8192, 128, False, "paged"),
]
BENCH_PAGE_SIZE = 256
_ratios = collections.defaultdict(float)
_POISON = (float("nan"), float("inf"), float("-inf"), 65504.0)
SENT_BF16 = 0x7FC1   # a bf16 NaN the kernel never writes


def label(key):
    if key[0] == "merge":
        return f"merge_attn_states of two halves, D{key[1]}"
    kind, ds, bn, wg, causal, split, tiling = key[:7]
    flags = [f for f, on in (("causal", causal), ("split", split)) if on]
    return f"{kind} <{','.join([str(ds), str(bn), str(wg)] + flags)}> {tiling}" + (f" page{key[7]}" if len(key) > 7
                                                                                    else "")


@pytest.fixture(scope="module", autouse=True)
def _report():
    t0 = time.time()
    yield
    if _ratios:
        print("\nlargest |err| / bound per path (attn_bf16_ref.o_bound / lse_bound / combine_bound):")
        for key in sorted({k for k, _ in _ratios}, key=str):
            print(f"  {label(key):<44} O {_ratios[(key, 'O')]:.3f}  lse {_ratios[(key, 'lse')]:.3f}")
    print(f"module time {time.time() - t0:.1f} s")


def _bf(*xs):
    return [x.to(torch.bfloat16) for x in xs]


def _guarded(shape, dtype):
    n = int(np.prod(shape))
    buf = torch.empty(n + 2 * MARGIN, dtype=dtype, device="cuda")
    if dtype == torch.bfloat16:
        buf.view(torch.int16).fill_(SENT_BF16)
    else:
        buf.view(torch.int32).fill_(SENT32)
    return buf, buf[MARGIN:MARGIN + n].view(shape)


def _margins_ok(buf, what):
    if buf.dtype == torch.bfloat16:
        bits = buf.view(torch.int16)
        assert bool((bits[:MARGIN] == SENT_BF16).all()), f"{what}: store before the output"
        assert bool((bits[-MARGIN:] == SENT_BF16).all()), f"{what}: store past the output"
    else:
        _assert_margins(buf, what)


def _guarded_call(fn, q):
    obuf, o = _guarded(tuple(q.shape), torch.bfloat16)
    lbuf, lse = _guarded(tuple(q.shape[:3]), torch.float32)
    torch.cuda.synchronize()
    n0 = _capi.launch_count()
    fn(o, lse)
    n = _capi.launch_count() - n0
    torch.cuda.synchronize()
    _margins_ok(obuf, "O")
    _margins_ok(lbuf, "lse")
    return o, lse, n


def paginate(k, v, lk, page_size, max_pages, poison, seed):
    """bf16 pools [num_pages, page_size, Hkv, D] holding k, v in randomly placed pages, unused pages `poison`, and the
    table [B, max_pages] padded with -1 past each sequence's pages."""
    B, Hkv, _, D = k.shape
    used = [-(-x // page_size) for x in lk]
    n_used = sum(used)
    num_pages = n_used + max(4, n_used // 4)
    perm = torch.randperm(num_pages, generator=torch.Generator().manual_seed(seed))
    pools = [torch.full((num_pages, page_size, Hkv, D), poison, dtype=k.dtype, device="cuda") for _ in range(2)]
    table = torch.full((B, max_pages), -1, dtype=torch.int32)
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


def _check_fp64(key, o, lse, q0, k0, v0, causal, splits, lq, lk, D, exact, what):
    sc, poly = R.kernel_scale(D), D <= 128
    if splits > 1:
        parts = S.part_references(q0, k0, v0, sc, causal, splits, lq, lk, exact)
        want_o, want_l, empty, ob, lb = BF.combine_bound(parts, poly)
    else:
        ref = S.reference(q0, k0, v0, sc, causal, lq, lk, exact)
        _, ob = BF.o_bound(ref, poly)
        want_o, want_l, empty, lb = ref["o"], ref["lse"], ref["empty"], BF.lse_bound(ref, poly)
    _check(key, (o, lse), (want_o, want_l), (ob, lb), empty, what)


def _same(a, b):
    return torch.equal(a.nan_to_num(1.0), b.nan_to_num(1.0)) and torch.equal(a.isnan(), b.isnan())


def _seqlens(q, k, v, causal, splits, lq, lk):
    return _guarded_call(lambda o, lse: flash_attn.fmha_fwd(q, k, v, o, lse=lse, causal=causal, num_splits=splits,
                                                            seqlens_q=lq, seqlens_k=lk), q)


def _paged(q, kp, vp, table, causal, splits, lq, lk):
    return _guarded_call(lambda o, lse: flash_attn.fmha_fwd(q, kp, vp, o, lse=lse, causal=causal, num_splits=splits,
                                                            seqlens_q=lq, seqlens_k=lk, block_table=table), q)


def _dense(q, k, v, causal, splits):
    return _guarded_call(lambda o, lse: flash_attn.fmha_fwd(q, k, v, o, lse=lse, causal=causal, num_splits=splits), q)


def _resolved(c, B):
    return c.splits if c.splits else _capi.lib().b200_fmha_fwd_f16_gqa_splits(B, c.H, c.Hkv, c.Nq, c.Nk, c.D)


@pytest.mark.parametrize("i", range(len(BF.CASES)), ids=lambda i: f"{BF.CASES[i][0]}{i}-D{BF.CASES[i][1].D}")
def test_case(i):
    kind, c = BF.CASES[i]
    for j, gen in enumerate(c.gens):
        poison = _POISON[(i + j) % len(_POISON)]
        if kind == "dense":
            B = 2
            splits = _resolved(c, B)
            key, launches = BF.path("dense", B, c.H, c.Hkv, c.Nq, c.Nk, c.D, c.causal, splits)
            what = f"{label(key)}: dense H{c.H} Hkv{c.Hkv} Nq{c.Nq} Nk{c.Nk} D{c.D} splits={c.splits} {gen}"
            q, k, v = _bf(*_inputs(gen, B, c.H, c.Hkv, c.Nq, c.Nk, c.D, None, seed=6131 * i + j))
            qc, kc, vc = q.clone(), k.clone(), v.clone()
            o, lse, n = _dense(q, k, v, c.causal, c.splits)
            assert n == launches, f"{what}: {n} launches, the path has {launches}"
            assert _same(q, qc) and _same(k, kc) and _same(v, vc), what + ": an input changed"
            _check_fp64(key, o, lse, q, k, v, c.causal, splits, [c.Nq] * B, [c.Nk] * B, c.D, BF.exact_scores(gen),
                        what)
            if c.Hkv < c.H:
                G = c.H // c.Hkv
                a = _dense(q, k, v, c.causal, 1)[:2]
                e = _dense(q, SR.expand(k, G).contiguous(), SR.expand(v, G).contiguous(), c.causal, 1)[:2]
                assert torch.equal(a[0], e[0]) and torch.equal(a[1], e[1]), what + ": GQA differs from repeated heads"
            continue
        B = len(c.lq)
        Nk = c.page_size * c.max_pages if kind == "paged" else c.Nk
        key, launches = BF.path(kind, B, c.H, c.Hkv, c.Nq, Nk, c.D, c.causal, c.splits,
                                getattr(c, "page_size", None))
        what = f"{label(key)}: H{c.H} Hkv{c.Hkv} Nq{c.Nq} Nk{Nk} D{c.D} splits={c.splits} {gen} pad={poison}"
        q0, k0, v0 = _bf(*_inputs(gen, B, c.H, c.Hkv, c.Nq, Nk, c.D, None, seed=7717 * i + j))
        q, k, v = _poison(q0, k0, v0, c.lq, c.lk, poison)
        lq, lk = _lens(c.lq), _lens(c.lk)
        if kind == "paged":
            kp, vp, table = paginate(k, v, c.lk, c.page_size, c.max_pages, poison, seed=31 * i + j)
            kc, vc, qc = kp.clone(), vp.clone(), q.clone()
            o, lse, n = _paged(q, kp, vp, table, c.causal, c.splits, lq, lk)
            assert _same(kp, kc) and _same(vp, vc) and _same(q, qc), what + ": an input changed"
            so, sl, _ = _seqlens(q, P.gather(kp, table, c.lk, Nk), P.gather(vp, table, c.lk, Nk), c.causal, c.splits,
                                 lq, lk)
            assert torch.equal(o, so) and torch.equal(lse, sl), what + ": not bitwise the seqlens call on the gathered cache"
        else:
            qc, kc, vc = q.clone(), k.clone(), v.clone()
            o, lse, n = _seqlens(q, k, v, c.causal, c.splits, lq, lk)
            assert _same(q, qc) and _same(k, kc) and _same(v, vc), what + ": an input changed"
            if c.splits == 1:
                for b in range(B):
                    if c.lq[b] < 1 or c.lk[b] < 1:
                        continue
                    qs = q[b:b + 1, :, :c.lq[b]].contiguous()
                    ks, vs = k[b:b + 1, :, :c.lk[b]].contiguous(), v[b:b + 1, :, :c.lk[b]].contiguous()
                    os_, ls, _ = _dense(qs, ks, vs, c.causal, 1)
                    assert torch.equal(o[b:b + 1, :, :c.lq[b]], os_) and torch.equal(lse[b:b + 1, :, :c.lq[b]], ls), \
                        f"{what}: sequence {b} is not bitwise the call on that sequence alone"
        assert n == launches, f"{what}: {n} launches, the path has {launches}"
        _check_fp64(key, o, lse, q0, k0, v0, c.causal, c.splits, c.lq, c.lk, c.D, BF.exact_scores(gen), what)


@pytest.mark.parametrize("splits", [1, 3])
def test_values_outside_fp16_range(splits):
    """V entries of 1e6 and 1e-30 and Q, K around 3e4 (scores finite in fp32): fp16 would overflow or flush them."""
    B, H, Hkv, Nq, Nk, D = 2, 8, 2, 64, 300, 128
    g = torch.Generator(device="cuda").manual_seed(41 + splits)
    q = (3e4 + 100 * torch.randn(B, H, Nq, D, device="cuda", generator=g)).to(torch.bfloat16)
    k = (3e4 * torch.randn(B, Hkv, Nk, D, device="cuda", generator=g).sign()
         + 100 * torch.randn(B, Hkv, Nk, D, device="cuda", generator=g)).to(torch.bfloat16)
    v = torch.randn(B, Hkv, Nk, D, device="cuda", generator=g)
    v[..., 0::2] *= 1e6
    v[..., 1::2] *= 1e-30
    v = v.to(torch.bfloat16)
    scale = 1e-9   # scores q.k ~ 1e10 in fp32, ~10 nats apart after the scale
    o, lse, n = _guarded_call(lambda o, lse: flash_attn.fmha_fwd(q, k, v, o, lse=lse, num_splits=splits, scale=scale),
                              q)
    assert n == 1 + (splits > 1)
    key = BF.path("dense", B, H, Hkv, Nq, Nk, D, False, splits)[0]
    sc = float(np.float32(scale))
    if splits > 1:
        parts = SR.part_references(q, k, v, sc, False, splits)
        want_o, want_l, empty, ob, lb = BF.combine_bound(parts, True)
    else:
        ref = SR.masked_reference(q, SR.expand(k, H // Hkv), SR.expand(v, H // Hkv), sc,
                                  torch.ones(Nq, Nk, dtype=torch.bool, device="cuda"))
        want_o, want_l, empty, ob, lb = ref["o"], ref["lse"], ref["empty"], BF.o_bound(ref, True)[1], \
            BF.lse_bound(ref, True)
    assert float(want_o[..., 0::2].abs().max()) > 1e5 and float(want_o[..., 1::2].abs().max()) < 1e-25
    assert float(q.float().abs().min()) > 65504 / 4 and float(v.float().abs().max()) > 65504
    _check(key, (o, lse), (want_o, want_l), (ob, lb), empty, f"outside fp16 range, splits={splits}")
    assert bool((o[..., 1::2] != 0).any()), "1e-30 outputs flushed to zero"


@pytest.mark.parametrize("splits", [1, 4], ids=["unsplit", "split"])
def test_graph_replay_with_new_lengths_and_tables(splits):
    B, H, Hkv, Nq, ps, maxp, D = 6, 16, 4, 1, 16, 128, 128
    q, k, v = _bf(*_inputs("randn", B, H, Hkv, Nq, ps * maxp, D, None, seed=11))
    kp, vp, table = paginate(k, v, [ps * maxp] * B, ps, maxp, float("nan"), seed=12)
    lq, lk = _lens([1] * B), _lens([5, 2048, 64, 0, 1000, 129])
    o, lse = torch.empty_like(q), torch.empty(q.shape[:3], device="cuda")
    call = lambda: flash_attn.fmha_fwd(q, kp, vp, o, lse=lse, num_splits=splits, seqlens_q=lq, seqlens_k=lk,
                                       block_table=table)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        call()
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        call()
    base = table.clone()
    for shift, new_k in ((1, [2048, 1, 0, 700, 63, 65]), (3, [100, 200, 300, 400, 500, 600])):
        table.copy_(base.roll(shift, 0))
        lk.copy_(_lens(new_k))
        graph.replay()
        torch.cuda.synchronize()
        eo, el, _ = _paged(q, kp, vp, table, False, splits, lq, lk)
        assert torch.equal(o, eo) and torch.equal(lse, el), f"graph replay with table shift {shift} differs from eager"


@pytest.mark.parametrize("D", [64, 128, 256])
def test_key_halves_merge_in_bf16(D):
    """Attention over keys [0, 512) and over [512, 1024), each with its lse, merged by merge_attn_states in bf16,
    against the full call's fp64 reference: the weighted part bounds (bf16 O), their lse errors through the weights,
    the merge's fp32 arithmetic and its rounding to bf16 (test_attn_causal_gpu's chunked-prefill bound with u = 2^-8)."""
    H, Nq, Nk, half = 4, 256, 1024, 512
    g = torch.Generator(device="cuda").manual_seed(17 + D)
    q, k, v = (torch.randn(1, H, n, D, device="cuda", generator=g).to(torch.bfloat16) for n in (Nq, Nk, Nk))
    sc, poly = R.kernel_scale(D), D <= 128
    parts = []
    for ks in (slice(0, half), slice(half, Nk)):
        kp, vp = k[:, :, ks].contiguous(), v[:, :, ks].contiguous()
        o, lse, _ = _dense(q, kp, vp, False, 1)
        parts.append((o, lse, R.reference(q, kp, vp, sc)))
    ref = R.reference(q, k, v, sc)
    merged = torch.empty(Nq, H, D, device="cuda", dtype=torch.bfloat16)
    merged_lse = torch.empty(H, Nq, device="cuda")
    (oa, la, ra), (ob, lb_, rb) = parts
    MA.merge_attn_states_cuda(merged, oa[0].transpose(0, 1).contiguous(), la[0].contiguous(),
                              ob[0].transpose(0, 1).contiguous(), lb_[0].contiguous(), merged_lse)
    torch.cuda.synchronize()
    wa = 1.0 / (1.0 + torch.exp(rb["lse"] - ra["lse"]))[..., None]
    wb = 1.0 - wa
    ba, bb = BF.o_bound(ra, poly)[1], BF.o_bound(rb, poly)[1]
    dl = (BF.lse_bound(ra, poly) + BF.lse_bound(rb, poly))[..., None]
    bound = (wa * ba + wb * bb + wa * wb * dl * (ra["o"] - rb["o"]).abs()
             + 2.0 ** -20 * (wa * ra["o"].abs() + wb * rb["o"].abs()) + BF.U8 * ref["o"].abs() + BF.O_FLOOR)
    err = (merged.double() - ref["o"][0].transpose(0, 1)).abs()
    bound = bound[0].transpose(0, 1)
    key = ("merge", D)
    _ratios[(key, "O")] = max(_ratios[(key, "O")], (err / bound).max().item())
    assert bool((err <= bound).all()), (err / bound).max().item()
    lse_err = (merged_lse.double() - ref["lse"][0]).abs()
    assert bool((lse_err <= BF.lse_bound(ref, poly)[0] + BF.lse_bound(ra, poly)[0] + BF.lse_bound(rb, poly)[0]
                 + 2.0 ** -20).all())


def _bench_lengths(index):
    """The seeded length draws of tools/bench_attn_bf16.py up to shape `index`."""
    rng = np.random.default_rng(0)
    lk = None
    for name, B, _, _, _, Nk, _, _, kind in BENCH_SHAPES[:index + 1]:
        lk = [int(x) for x in rng.integers(256, 8192 + 1, size=B)] if kind in ("seqlens", "paged") else [Nk] * B
    return lk


def _sampled_rows(lq, lk, D, causal):
    if lq <= 16:
        return list(range(lq))
    kbn, _ = M.kernel_shape(D)
    rows = {0, 63, 64, 127, 128, lq - 1, lq - 2}
    rows |= {i for i in range(lq) if causal and (i + lk - lq) % kbn in (0, kbn - 1)}
    return sorted(r for r in rows if 0 <= r < lq)[:48]


@pytest.mark.parametrize("index", range(len(BENCH_SHAPES)), ids=lambda i: BENCH_SHAPES[i][0].replace(" ", "-") + str(i))
def test_benchmarked_shape(index):
    """Every shape of tools/bench_attn_bf16.py at full size: sampled rows of three sequences within the fp64 bound
    (whole rows of the split parts when the call splits); paged bit for bit the seqlens call on the gathered cache."""
    name, B, H, Hkv, Nq, Nk, D, causal, kind = BENCH_SHAPES[index]
    lk = _bench_lengths(index)
    lq = [Nq] * B
    g = torch.Generator(device="cuda").manual_seed(300 + index)
    q = torch.randn(B, H, Nq, D, device="cuda", generator=g).to(torch.bfloat16)
    k = torch.randn(B, Hkv, Nk, D, device="cuda", generator=g).to(torch.bfloat16)
    v = torch.randn(B, Hkv, Nk, D, device="cuda", generator=g).to(torch.bfloat16)
    tq, tk = _lens(lq), _lens(lk)
    splits_arg = 1 if kind == "dense" else 0
    splits = 1 if kind == "dense" else _capi.lib().b200_fmha_fwd_f16_gqa_splits(B, H, Hkv, Nq, Nk, D)
    if kind == "dense":
        o, lse, n = _dense(q, k, v, causal, 1)
    elif kind == "decode":
        o, lse, n = _dense(q, k, v, causal, 0)
    elif kind == "seqlens":
        o, lse, n = _seqlens(q, k, v, causal, 0, tq, tk)
    else:
        kp, vp, table = paginate(k, v, lk, BENCH_PAGE_SIZE, Nk // BENCH_PAGE_SIZE, float("nan"), seed=index)
        o, lse, n = _paged(q, kp, vp, table, causal, 0, tq, tk)
        so, sl, _ = _seqlens(q, k, v, causal, 0, tq, tk)
        assert torch.equal(o, so) and torch.equal(lse, sl), f"{name}: not bitwise the seqlens call"
        del kp, vp, table
    assert n == 1 + (splits > 1)
    key = BF.path("paged" if kind == "paged" else "seqlens", B, H, Hkv, Nq, Nk, D, causal, splits,
                  BENCH_PAGE_SIZE)[0]
    sc, poly = R.kernel_scale(D), D <= 128
    G = H // Hkv
    for b in sorted({int(np.argmin(lk)), int(np.argmax(lk)), B // 2}):
        what = f"{name} sequence {b} (Lq {lq[b]}, Lk {lk[b]}) splits={splits_arg}"
        qb, kb, vb = q[b:b + 1], k[b:b + 1, :, :lk[b]], v[b:b + 1, :, :lk[b]]
        if splits > 1:
            _check_fp64(key, o[b:b + 1], lse[b:b + 1], qb, kb, vb, causal, splits, [lq[b]], [lk[b]], D, False, what)
            continue
        r = torch.tensor(_sampled_rows(lq[b], lk[b], D, causal), device="cuda")
        i, j = r[:, None], torch.arange(lk[b], device="cuda")[None, :]
        vis = (j <= i + (lk[b] - lq[b])) if causal else torch.ones_like(i * j, dtype=torch.bool)
        ref = SR.masked_reference(qb[:, :, r], SR.expand(kb, G), SR.expand(vb, G), sc, vis[None, None])
        _check(key, (o[b:b + 1, :, r], lse[b:b + 1, :, r]), (ref["o"], ref["lse"]),
               (BF.o_bound(ref, poly)[1], BF.lse_bound(ref, poly)), ref["empty"], what)
    del q, k, v, o, lse
    torch.cuda.empty_cache()


def test_sdpa_bf16():
    B, H, Hkv, Nq, Nk, D = 2, 8, 2, 130, 500, 128
    q, k, v = _bf(*_inputs("randn", B, H, Hkv, Nq, Nk, D, None, seed=19))
    o, _, _ = _dense(q, k, v, False, 1)
    ref = torch.nn.functional.scaled_dot_product_attention(q, k, v, enable_gqa=True)
    assert (o.float() - ref.float()).abs().max().item() < 2e-2


# ------------------------------------------------------------------ kernel names
# torch.profiler runs in a child process.  In one process, a profiler session followed by many launches leaves later
# sessions without CUDA records (see test_attn_paged_gpu.test_kernel_names), and this module runs before the fp16
# modules whose kernel-name tests rely on being the first sessions of the process.  The child runs every case in one
# session (test_attn_seqlens_gpu._kernels_per_call) and reports the names; the parent process never starts the profiler.
def _case_call(i):
    """(path key, a call of case i on fresh randn inputs, description)."""
    kind, c = BF.CASES[i]
    if kind == "dense":
        B = 2
        key = BF.path("dense", B, c.H, c.Hkv, c.Nq, c.Nk, c.D, c.causal, _resolved(c, B))[0]
        q, k, v = _bf(*_inputs("randn", B, c.H, c.Hkv, c.Nq, c.Nk, c.D, None, seed=i))
        o = torch.empty_like(q)
        fn = lambda: flash_attn.fmha_fwd(q, k, v, o, causal=c.causal, num_splits=c.splits)
    else:
        B = len(c.lq)
        Nk = c.page_size * c.max_pages if kind == "paged" else c.Nk
        key = BF.path(kind, B, c.H, c.Hkv, c.Nq, Nk, c.D, c.causal, c.splits, getattr(c, "page_size", None))[0]
        q, k, v = _bf(*_inputs("randn", B, c.H, c.Hkv, c.Nq, Nk, c.D, None, seed=i))
        lq, lk, o = _lens(c.lq), _lens(c.lk), torch.empty_like(q)
        extra = {}
        if kind == "paged":
            k, v, table = paginate(k, v, c.lk, c.page_size, c.max_pages, 0.0, seed=i)
            extra = dict(block_table=table)
        fn = lambda: flash_attn.fmha_fwd(q, k, v, o, causal=c.causal, num_splits=c.splits, seqlens_q=lq, seqlens_k=lk,
                                         **extra)
    return key, fn, f"{label(key)}: {kind} H{c.H} Hkv{c.Hkv} Nq{c.Nq} D{c.D} splits={c.splits}"


def _profile_all_cases():
    """Child process: the CUDA kernel names of every case under torch.profiler, as one JSON line on stdout."""
    fns = [_case_call(i)[1] for i in range(len(BF.CASES))]
    print("KERNEL_NAMES " + json.dumps(_kernels_per_call(fns)))


@pytest.fixture(scope="module")
def profiled_names():
    tests = Path(__file__).resolve().parent
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([str(tests.parent), str(tests)]
                                                      + [p for p in [os.environ.get("PYTHONPATH")] if p]))
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [
        "-c", "import test_attn_bf16_gpu as T; T._profile_all_cases()"]
    r = subprocess.run(cmd, cwd=tests.parent, env=env, capture_output=True, text=True, timeout=900)
    lines = [x for x in r.stdout.splitlines() if x.startswith("KERNEL_NAMES ")]
    assert r.returncode == 0 and lines, f"profiling child failed ({r.returncode}):\n{r.stdout[-2000:]}{r.stderr[-4000:]}"
    return json.loads(lines[-1][len("KERNEL_NAMES "):])


@pytest.mark.parametrize("i", range(len(BF.CASES)), ids=lambda i: f"{BF.CASES[i][0]}{i}-D{BF.CASES[i][1].D}")
def test_kernel_names(profiled_names, i):
    key, _, what = _case_call(i)
    names = profiled_names[i]
    assert names, what + ": the profiler recorded no kernel"
    assert BF.parse_instantiations(names) == [BF.instantiation(key)], f"{what}: ran {names}"
    assert not S.parse_instantiations(names) and not P.parse_instantiations(names), f"{what}: ran {names}"
    assert not any("attn_fwd_kernel<" in s for s in names), f"{what}: ran {names}"
    assert sum("attn_combine_kernel" in s for s in names) == int(key[5]), f"{what}: ran {names}"
