"""Per-sequence query and key lengths (b200_fmha_fwd_f16_seqlens, flash_attn.fmha_fwd(seqlens_q=, seqlens_k=)) on the
GPU, over every path of attn_seqlens_ref.CASES_BY_SHAPE.

Every case mixes the lengths of its sequences and poisons what lies past them: K / V rows >= Lk_b hold NaN, +Inf, -Inf
or 65504 (in turn over the generators), Q rows >= Lq_b hold NaN, and O / lse sit inside NaN guard bands.  Checked:
  * the fp64 reference with each sequence's visibility (attn_ref.o_bound / lse_bound unsplit, attn_split_ref's
    combine_bound of the restated per-sequence split ranges split); padded rows and rows without a key exactly O = 0,
    lse = -inf; the inputs come back unchanged;
  * unsplit: every sequence's rows bit for bit fmha_fwd on that sequence alone (Nq = Lq_b, Nk = Lk_b);
  * full-length arrays: bit for bit the call without lengths, split or not;
  * _capi.launch_count() up by 1 unsplit, 2 split; under torch.profiler (in a child process) the restated
    attn_fwd_seqlens_kernel<...>, the combine exactly when it splits.
Then clamping, CUDA graphs and a side stream, a 65536-key sequence among short ones, and SDPA with an explicit mask.
The largest |err| / bound per path is printed at the end of the module (pytest -s).
"""
import collections
import math
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from torch.profiler import ProfilerActivity, profile

import attn_mask_ref as M
import attn_ref as R
import attn_seqlens_ref as S
import attn_split_ref as SR
from leetcuda_b200 import _capi, flash_attn
from test_attn_gqa_gpu import _inputs
from test_attn_numerics_gpu import _assert_margins, _guarded

pytestmark = pytest.mark.gpu

_ratios = collections.defaultdict(float)
_POISON = (float("nan"), float("inf"), float("-inf"), 65504.0)


def label(key):
    ds, bn, wg, causal, split, tiling = key
    flags = [f for f, on in (("causal", causal), ("split", split)) if on]
    return f"<{','.join([str(ds), str(bn), str(wg)] + flags)}> {tiling}"


@pytest.fixture(scope="module", autouse=True)
def _report():
    t0 = time.time()
    yield
    if _ratios:
        print("\nlargest |err| / bound per path (attn_ref.o_bound / lse_bound, attn_split_ref.combine_bound):")
        for key in sorted({k for k, _ in _ratios}):
            print(f"  {label(key):<32} O {_ratios[(key, 'O')]:.3f}  lse {_ratios[(key, 'lse')]:.3f}")
    print(f"module time {time.time() - t0:.1f} s")


def _lens(x):
    return torch.tensor(list(x), dtype=torch.int32, device="cuda")


def _call(q, k, v, o, lse, causal, splits, lq, lk):
    flash_attn.fmha_fwd(q, k, v, o, lse=lse, causal=causal, num_splits=splits, seqlens_q=lq, seqlens_k=lk)


def _run(q, k, v, causal, splits, lq, lk):
    obuf, o = _guarded(tuple(q.shape), torch.float16)
    lbuf, lse = _guarded(tuple(q.shape[:3]), torch.float32)
    torch.cuda.synchronize()
    n0 = _capi.launch_count()
    _call(q, k, v, o, lse, causal, splits, lq, lk)
    n = _capi.launch_count() - n0
    torch.cuda.synchronize()
    _assert_margins(obuf, "O")
    _assert_margins(lbuf, "lse")
    return o, lse, n


def _poison(q, k, v, lq, lk, value):
    q, k, v = q.clone(), k.clone(), v.clone()
    for b in range(q.shape[0]):
        q[b, :, lq[b]:] = float("nan")
        k[b, :, lk[b]:] = value
        v[b, :, lk[b]:] = value
    return q, k, v


def _kernels_per_call(fns):
    """[names of the CUDA kernels fn launches for fn in fns] from one torch.profiler session.  On an H100, a process that
    had run some 30 short sessions recorded later ones without some or all of their kernels; a single session for all calls
    does not depend on that.  The calls run one after another on a synchronised device, and the records split at a
    marker kernel (torch.cuda._sleep) launched before every call and after the last."""
    out = []
    for _ in range(3):
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            time.sleep(0.002)
            for fn in fns:
                torch.cuda._sleep(1)
                fn()
                torch.cuda.synchronize()
            torch.cuda._sleep(1)
            torch.cuda.synchronize()
            time.sleep(0.002)
        names = [e.name for e in sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA),
                                        key=lambda e: e.time_range.start)]
        out = []
        for name in names:
            if name == names[0]:
                out.append([])
            else:
                out[-1].append(name)
        out = out[:-1]
        if len(out) == len(fns) and names.count(names[0]) == len(fns) + 1:
            return out
    return out


def _profile_all_cases():
    """Child process: the CUDA kernel names of every case, as one JSON line on stdout."""
    import json
    fns = []
    for i, c in enumerate(S.CASES_BY_SHAPE):
        q, k, v = _inputs("randn", len(c.lq), c.H, c.Hkv, c.Nq, c.Nk, c.D, None, seed=i)
        lq, lk, o = _lens(c.lq), _lens(c.lk), torch.empty_like(q)
        fns.append(lambda q=q, k=k, v=v, o=o, c=c, lq=lq, lk=lk: _call(q, k, v, o, None, c.causal, c.splits, lq, lk))
    print("KERNEL_NAMES " + json.dumps(_kernels_per_call(fns)))


def profiled_names_of(module):
    """Run module._profile_all_cases() in a child process and return what it reports."""
    import json
    import os
    import subprocess
    import sys
    from pathlib import Path
    tests = Path(__file__).resolve().parent
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([str(tests.parent), str(tests)]
                                                      + [p for p in [os.environ.get("PYTHONPATH")] if p]))
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [
        "-c", f"import {module} as T; T._profile_all_cases()"]
    r = subprocess.run(cmd, cwd=tests.parent, env=env, capture_output=True, text=True, timeout=900)
    lines = [x for x in r.stdout.splitlines() if x.startswith("KERNEL_NAMES ")]
    assert r.returncode == 0 and lines, f"profiling child failed ({r.returncode}):\n{r.stdout[-2000:]}{r.stderr[-4000:]}"
    return json.loads(lines[-1][len("KERNEL_NAMES "):])


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


@pytest.mark.parametrize("i", range(len(S.CASES_BY_SHAPE)), ids=lambda i: f"case{i}-D{S.CASES_BY_SHAPE[i].D}")
def test_case_against_fp64(i):
    c = S.CASES_BY_SHAPE[i]
    B = len(c.lq)
    key, launches = S.path(B, c.H, c.Hkv, c.Nq, c.Nk, c.D, c.causal, c.splits)
    G, poly, sc = c.H // c.Hkv, c.D <= 128, R.kernel_scale(c.D)
    lq, lk = _lens(c.lq), _lens(c.lk)
    for j, gen in enumerate(c.gens):
        poison = _POISON[(i + j) % len(_POISON)]
        what = f"{label(key)}: H{c.H} Hkv{c.Hkv} Nq{c.Nq} Nk{c.Nk} D{c.D} splits={c.splits} {gen} pad={poison}"
        q0, k0, v0 = _inputs(gen, B, c.H, c.Hkv, c.Nq, c.Nk, c.D, None, seed=7717 * i + j)
        q, k, v = _poison(q0, k0, v0, c.lq, c.lk, poison)
        qc, kc, vc = q.clone(), k.clone(), v.clone()
        o, lse, n = _run(q, k, v, c.causal, c.splits, lq, lk)
        assert n == launches, f"{what}: {n} launches, the path has {launches}"
        for a, b in ((q, qc), (k, kc), (v, vc)):
            assert torch.equal(a.nan_to_num(1.0), b.nan_to_num(1.0)) and torch.equal(a.isnan(), b.isnan()), \
                what + ": an input changed"
        exact = M.exact_scores(gen)
        if c.splits > 1:
            parts = S.part_references(q0, k0, v0, sc, c.causal, c.splits, c.lq, c.lk, exact)
            want_o, want_l, empty, ob, lb = SR.combine_bound(parts, poly)
        else:
            ref = S.reference(q0, k0, v0, sc, c.causal, c.lq, c.lk, exact)
            _, ob = R.o_bound(ref, poly)
            want_o, want_l, empty, lb = ref["o"], ref["lse"], ref["empty"], R.lse_bound(ref, poly)
        _check(key, (o, lse), (want_o, want_l), (ob, lb), empty, what)

        if c.splits == 1:
            for b in range(B):
                if c.lq[b] < 1 or c.lk[b] < 1:
                    continue
                qs = q[b:b + 1, :, :c.lq[b]].contiguous()
                ks, vs = k[b:b + 1, :, :c.lk[b]].contiguous(), v[b:b + 1, :, :c.lk[b]].contiguous()
                os_, ls = torch.empty_like(qs), torch.empty(qs.shape[:3], device="cuda")
                flash_attn.fmha_fwd(qs, ks, vs, os_, lse=ls, causal=c.causal, num_splits=1)
                torch.cuda.synchronize()
                assert torch.equal(o[b:b + 1, :, :c.lq[b]], os_) and torch.equal(lse[b:b + 1, :, :c.lq[b]], ls), \
                    f"{what}: sequence {b} is not bitwise the call on that sequence alone"
        if j == 0:
            full_q, full_k = _lens([c.Nq] * B), _lens([c.Nk] * B)
            fo, fl, _ = _run(q0, k0, v0, c.causal, c.splits, full_q, full_k)
            go, gl = torch.empty_like(fo), torch.empty_like(fl)
            flash_attn.fmha_fwd(q0, k0, v0, go, lse=gl, causal=c.causal, num_splits=c.splits)
            torch.cuda.synchronize()
            assert torch.equal(fo, go) and torch.equal(fl, gl), what + ": full lengths differ from the call without"


# torch.profiler runs in a child process, all cases in one session; this process never starts it (see
# _kernels_per_call, and test_attn_bf16_gpu: the fp16 modules that sort after this one rely on the first sessions).
@pytest.fixture(scope="module")
def profiled_names():
    return profiled_names_of("test_attn_seqlens_gpu")


@pytest.mark.parametrize("i", range(len(S.CASES_BY_SHAPE)), ids=lambda i: f"case{i}-D{S.CASES_BY_SHAPE[i].D}")
def test_kernel_names(profiled_names, i):
    c = S.CASES_BY_SHAPE[i]
    key, _ = S.path(len(c.lq), c.H, c.Hkv, c.Nq, c.Nk, c.D, c.causal, c.splits)
    what = f"{label(key)}: H{c.H} Hkv{c.Hkv} Nq{c.Nq} Nk{c.Nk} D{c.D} splits={c.splits}"
    names = profiled_names[i] if i < len(profiled_names) else []
    assert names, what + ": the profiler recorded no kernel"
    assert S.parse_instantiations(names) == [S.instantiation(key)], f"{what}: ran {names}"
    assert not any("attn_fwd_kernel<" in s for s in names), f"{what}: ran {names}"
    assert sum("attn_combine_kernel" in s for s in names) == int(key[4]), f"{what}: ran {names}"


@pytest.mark.parametrize("splits", [1, 3])
def test_lengths_are_clamped(splits):
    B, H, Hkv, Nq, Nk, D = 4, 8, 2, 5, 300, 128
    q, k, v = _inputs("randn", B, H, Hkv, Nq, Nk, D, None, seed=5)
    raw_q, raw_k = [-3, 9, 5, 100000], [-1, 1000, 77, 2 ** 31 - 1]
    got = _run(q, k, v, True, splits, _lens(raw_q), _lens(raw_k))[:2]
    want = _run(q, k, v, True, splits, _lens(S.clamp(raw_q, Nq)), _lens(S.clamp(raw_k, Nk)))[:2]
    assert torch.equal(got[0], want[0]) and torch.equal(got[1], want[1])
    assert bool((got[0][0] == 0).all()) and bool((got[1][0] == -math.inf).all())


def test_null_length_arrays_mean_full():
    B, H, Hkv, Nq, Nk, D = 3, 8, 2, 130, 300, 64
    q, k, v = _inputs("randn", B, H, Hkv, Nq, Nk, D, None, seed=6)
    o1, l1, _ = _run(q, k, v, True, 1, _lens([Nq] * B), None)
    o2, l2, _ = _run(q, k, v, True, 1, None, _lens([Nk] * B))
    o3, l3 = torch.empty_like(o1), torch.empty_like(l1)
    flash_attn.fmha_fwd(q, k, v, o3, lse=l3, causal=True)
    torch.cuda.synchronize()
    assert torch.equal(o1, o3) and torch.equal(o2, o3) and torch.equal(l1, l3) and torch.equal(l2, l3)


# ------------------------------------------------------------------ graphs, streams, long sequences, SDPA
@pytest.mark.parametrize("splits", [1, 4], ids=["unsplit", "split"])
def test_graph_replay_with_new_lengths_and_side_stream(splits):
    B, H, Hkv, Nq, Nk, D = 6, 16, 4, 1, 2048, 128
    q, k, v = _inputs("randn", B, H, Hkv, Nq, Nk, D, None, seed=11)
    lq, lk = _lens([1] * B), _lens([5, 2048, 64, 0, 1000, 129])
    o, lse = torch.empty_like(q), torch.empty(q.shape[:3], device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(2):
            _call(q, k, v, o, lse, False, splits, lq, lk)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    eo, el, _ = _run(q, k, v, False, splits, lq, lk)
    assert torch.equal(o, eo) and torch.equal(lse, el), "side stream differs from eager"
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        _call(q, k, v, o, lse, False, splits, lq, lk)
    for new_k in ([2048, 1, 0, 700, 63, 65], [100, 200, 300, 400, 500, 600]):
        lk.copy_(_lens(new_k))
        graph.replay()
        torch.cuda.synchronize()
        eo, el, _ = _run(q, k, v, False, splits, lq, lk)
        assert torch.equal(o, eo) and torch.equal(lse, el), f"graph replay with lengths {new_k} differs from eager"


def test_long_sequence_among_short_ones():
    """One 65536-key sequence in a decode batch: the automatic split count follows the padded shape, so the short
    sequences' splits are mostly empty."""
    B, H, Hkv, Nq, Nk, D = 4, 8, 2, 1, 65536, 128
    q, k, v = _inputs("randn", B, H, Hkv, Nq, Nk, D, None, seed=13)
    lens_k = [65536, 3, 0, 700]
    q, k, v = _poison(q, k, v, [1] * B, lens_k, float("nan"))
    splits = _capi.lib().b200_fmha_fwd_f16_gqa_splits(B, H, Hkv, Nq, Nk, D)
    assert splits > 1
    o, lse, n = _run(q, k, v, False, 0, _lens([1] * B), _lens(lens_k))
    assert n == 2
    q0 = q.clone()
    k0, v0 = k.nan_to_num(0.0), v.nan_to_num(0.0)
    parts = S.part_references(q0, k0, v0, R.kernel_scale(D), False, splits, [1] * B, lens_k)
    want_o, want_l, empty, ob, lb = SR.combine_bound(parts, True)
    key = S.path(B, H, Hkv, Nq, Nk, D, False, splits)[0]
    _check(key, (o, lse), (want_o, want_l), (ob, lb), empty, "long sequence")


def test_sdpa_with_an_explicit_mask():
    B, H, Hkv, Nq, Nk, D = 3, 8, 2, 40, 500, 64
    q, k, v = _inputs("randn", B, H, Hkv, Nq, Nk, D, None, seed=17)
    lq, lk = [40, 7, 1], [500, 300, 9]
    o, _, _ = _run(q, k, v, True, 1, _lens(lq), _lens(lk))
    vis = torch.from_numpy(np.stack([S.visible(Nq, Nk, lq[b], lk[b], True) for b in range(B)])[:, None]).cuda()
    ref = F.scaled_dot_product_attention(q, k, v, attn_mask=vis, enable_gqa=True)
    for b in range(B):
        err = (o[b, :, :lq[b]].float() - ref[b, :, :lq[b]].float()).abs().max().item()
        assert err < 2e-3, (b, err)
        assert bool((o[b, :, lq[b]:] == 0).all())
